"""flax.nn-0.3.0-shaped model protocol over libsmd (what train_ncsn.py:193-203 and sample_ncsn.py:331-342 use):

    module = ncsn.TransformerDDPM.partial(num_layers=..., num_heads=..., num_mlp_layers=..., mlp_dims=...)
    _, params = module.init_by_shape(rng, [((B, *shape), float32), ((B, *[1]*len(shape)), float32)])
    model = nn.Model(module, params);   eps_hat = model(inputs, t);   model.params;   model.replace(params=...)

Parameters live in ONE flat fp32 device arena (torch tensor); ``model.params`` is a nested dict of views into it,
so all-reduce / clip / Adam are single fused passes.  Compute always goes through the C ABI (no CPU fallback).
"""
from __future__ import annotations

from typing import Dict, Optional, Sequence, Tuple

import numpy as np
import torch

from .engine import ARCHS, Engine, ModelConfig


class ModuleSpec:
    """A score-network class bound to its keyword arguments (what ``Module.partial(**kw)`` returns in flax.nn)."""

    def __init__(self, arch: str, **kwargs):
        if arch not in ARCHS:
            raise ValueError(f"unknown architecture {arch!r}")
        self.arch = arch
        # DenseDDPM accepts-and-ignores the transformer kwargs (SURVEY D5: train_ncsn.py:321-326 always passes them)
        self.kwargs = dict(kwargs)
        self._engines: list = []
        self.cta_group = 2

    def partial(self, **kwargs) -> "ModuleSpec":
        kw = dict(self.kwargs)
        kw.update(kwargs)
        return ModuleSpec(self.arch, **kw)

    def model_config(self, input_shape: Sequence[int]) -> ModelConfig:
        kw = self.kwargs
        dense = ARCHS[self.arch] in (1, 2)
        if dense:
            if len(input_shape) != 1:
                raise ValueError(f"{self.arch} expects inputs of shape (batch, z_dims)")
            # models/ncsn.py:125 signature default is 3; train_ncsn.py passes FLAGS.num_layers
            return ModelConfig(arch=self.arch, num_layers=int(kw.get("num_layers", 3)),
                               mlp_dims=int(kw.get("mlp_dims", 2048)), seq_len=1, channels=int(input_shape[-1]))
        if len(input_shape) != 2:
            raise ValueError(f"{self.arch} expects inputs of shape (batch, seq_len, channels)")
        extra = {}
        if self.arch == "TransformerMDN":   # models/autoregressive.py:40-47 keyword mdn_mixtures
            extra["mdn_components"] = int(kw.get("mdn_mixtures", 100))
        return ModelConfig(arch=self.arch, num_layers=int(kw.get("num_layers", 6)), num_heads=int(kw.get("num_heads", 8)),
                           num_mlp_layers=int(kw.get("num_mlp_layers", 2)), mlp_dims=int(kw.get("mlp_dims", 2048)),
                           seq_len=int(input_shape[0]), channels=int(input_shape[1]), **extra)

    def engine(self, input_shape, max_batch: int, training: bool) -> Engine:
        """Smallest cached engine of this spec that fits (shape, training, batch); created on demand."""
        shape = tuple(int(s) for s in input_shape)
        best = None
        for eng in self._engines:
            if eng._shape == shape and eng.training == bool(training) and eng.max_batch >= max_batch:
                if best is None or eng.max_batch < best.max_batch:
                    best = eng
        if best is None:
            best = Engine(self.model_config(shape), max_batch=max_batch, cta_group=self.cta_group, training=training)
            best._shape = shape
            self._engines.append(best)
        return best

    def init_by_shape(self, rng, input_specs, seed: Optional[int] = None):
        """Returns (None, params): flax-default initialisers (see Engine.init_params) seeded from the jax key."""
        (shape, _dtype) = input_specs[0]
        batch, input_shape = int(shape[0]), tuple(int(s) for s in shape[1:])
        eng = self.engine(input_shape, batch, training=False)
        if seed is None:
            k = np.asarray(rng, dtype=np.uint32).reshape(-1)
            seed = int(k[0]) * (1 << 32) + int(k[1]) if k.size >= 2 else int(k[0])
        flat = eng.init_params(seed=seed)
        return None, ParamArena(self, input_shape, flat)


class ParamArena:
    """Flat fp32 parameter arena + the layout that names its tensors."""

    def __init__(self, spec: ModuleSpec, input_shape, flat):
        self.spec = spec
        self.input_shape = tuple(input_shape)
        eng = spec.engine(self.input_shape, 1, training=False)
        self.layout = eng.layout
        if isinstance(flat, np.ndarray):
            flat = torch.from_numpy(np.ascontiguousarray(flat, np.float32))
        if torch.cuda.is_available() and not flat.is_cuda:
            flat = flat.cuda()
        self.flat = flat
        self.version = 0

    def bump(self) -> None:
        self.version += 1

    def as_dict(self) -> Dict[str, torch.Tensor]:
        out: Dict[str, torch.Tensor] = {}
        for name, off, shape in self.layout:
            n = int(np.prod(shape))
            out[name] = self.flat[off:off + n].view(*shape)
        return out

    def nested(self) -> dict:
        tree: dict = {}
        for name, t in self.as_dict().items():
            node = tree
            parts = name.split(".")
            for p in parts[:-1]:
                node = node.setdefault(p, {})
            node[parts[-1]] = t
        return tree

    def clone(self) -> "ParamArena":
        return ParamArena(self.spec, self.input_shape, self.flat.clone())


class Model:
    """nn.Model(module, params): a callable bound to its parameters."""

    def __init__(self, module: ModuleSpec, params: ParamArena):
        self.module = module
        self.arena = params

    @property
    def params(self) -> dict:
        return self.arena.nested()

    def replace(self, params=None) -> "Model":
        if params is None:
            return Model(self.module, self.arena)
        if isinstance(params, ParamArena):
            return Model(self.module, params)
        raise TypeError("replace(params=...) expects the ParamArena of another Model / EMA / optimizer target")

    def engine(self, batch: int, training: bool = False) -> Engine:
        eng = self.module.engine(self.arena.input_shape, batch, training)
        tag = (id(self.arena.flat), self.arena.version)
        if getattr(eng, "_packed_tag", None) != tag:
            eng.set_params(self.arena.flat)
            eng._packed_tag = tag
        return eng

    def __call__(self, inputs, t=None, shift=True):
        """Score networks: eps_hat = model(inputs, t).  TransformerMDN: (pi, mu, log_sigma) = model(inputs, shift)
        (models/autoregressive.py:40), the second positional argument being `shift`."""
        x = _as_device_f32(inputs)
        if self.module.arch == "TransformerMDN":
            return self.engine(x.shape[0]).mdn_forward(x, shift=bool(shift if t is None else t))
        if t is None:
            raise TypeError("model(inputs, t): the score networks need the noise level t")
        tt = _as_device_f32(t).reshape(-1)
        if tt.numel() != x.shape[0]:
            raise ValueError("t must have one entry per example (rank equal to inputs' rank in the reference)")
        return self.engine(x.shape[0]).forward(x, tt)


def _as_device_f32(a) -> torch.Tensor:
    if isinstance(a, torch.Tensor):
        t = a
    else:
        t = torch.from_numpy(np.ascontiguousarray(np.asarray(a), dtype=np.float32))
    if t.dtype != torch.float32:
        t = t.float()
    if not t.is_cuda:
        t = t.cuda()
    return t.contiguous()
