"""Host-side driver of libsmd: owns the plan, the device workspace and the flat fp32 parameter arena.

PyTorch is used only as the device-memory / stream provider; all compute goes through the C ABI
(include/smd.h).  Everything here raises if CUDA or libsmd.so is unavailable -- no CPU fallback.
"""
from __future__ import annotations

import ctypes as C
import os
from dataclasses import dataclass, asdict
from typing import Dict, List, Optional, Tuple

import numpy as np
import torch

from . import lib as _lib

ARCHS = {"TransformerDDPM": 0, "TransformerDDPM4": 0, "DenseDDPM": 1, "DenseNCSN": 2, "TransformerMDN": 3}
SEQUENCE_ARCHS = (0, 3)   # (B, S, C) inputs; the dense networks take (B, C)
PRECISIONS = {"bf16": 0, "bf16x3": 1}


@dataclass
class ModelConfig:
    """Keyword surface of the reference score networks (models/ncsn.py:125,141-147; train_ncsn.py:321-326)."""
    arch: str = "TransformerDDPM"
    num_layers: int = 6
    num_heads: int = 8
    num_mlp_layers: int = 2
    mlp_dims: int = 2048
    seq_len: int = 32
    channels: int = 42
    mdn_components: int = 100   # TransformerMDN only (train_mdn.py --mdn_components)

    def flops_fwd_per_sample(self) -> float:
        """Algorithmic forward FLOPs per sample (SURVEY section 8(d))."""
        E, S, C, M = 128, self.seq_len, self.channels, self.mlp_dims
        if ARCHS[self.arch] == 0:
            L, K = self.num_layers, self.num_mlp_layers
            mac_tok = C * E + L * (4 * E * E + 2 * S * E + 2 * E * M) + E * M + K * 2 * M * M + M * C
        else:
            K, S = self.num_layers, 1      # DenseDDPM: one (B, C) vector per example
            mac_tok = C * M + K * 2 * M * M + M * C
        mac_film = K * (128 * 512 + 512 * 512 + 2 * 512 * M)
        return 2.0 * (S * mac_tok + mac_film)


def _ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


def _f32c(t: torch.Tensor, name: str) -> torch.Tensor:
    if t.dtype != torch.float32 or not t.is_cuda or not t.is_contiguous():
        raise ValueError(f"{name} must be a contiguous float32 CUDA tensor")
    return t


class Engine:
    def __init__(self, cfg: ModelConfig, max_batch: int, cta_group: int = 2, training: bool = False,
                 device: Optional[str] = None, sampler_T: Optional[int] = None, precision: Optional[str] = None):
        if cfg.arch not in ARCHS:
            raise ValueError(f"unknown architecture {cfg.arch!r}")
        self.cfg = cfg
        self.max_batch = int(max_batch)
        self.lib = _lib.load_library()
        # "bf16" (default, the timed path) or "bf16x3" (strict: split operands, exact activations; forward only)
        precision = precision or os.environ.get("SMD_PRECISION", "bf16")
        if precision not in PRECISIONS:
            raise ValueError(f"unknown precision {precision!r} (expected one of {sorted(PRECISIONS)})")
        self.precision = precision
        self.mdn = ARCHS[cfg.arch] == 3
        if sampler_T is None:
            sampler_T = 0 if training or self.mdn else 1000
        c = _lib.SmdConfig(ARCHS[cfg.arch], cfg.num_layers, cfg.num_heads, cfg.num_mlp_layers, cfg.mlp_dims,
                           cfg.seq_len if ARCHS[cfg.arch] in SEQUENCE_ARCHS else 1, cfg.channels, self.max_batch,
                           int(cta_group), int(training), int(sampler_T), PRECISIONS[precision])
        h = C.c_void_p()
        if self.mdn:
            _lib.check(self.lib.smd_mdn_plan_create(C.byref(c), int(cfg.mdn_components), C.byref(h)))
        else:
            _lib.check(self.lib.smd_plan_create(C.byref(c), C.byref(h)))
        self._plan = h
        self._comm_stream = None
        self.seq_len = cfg.seq_len if ARCHS[cfg.arch] in SEQUENCE_ARCHS else 1
        self.training = bool(training)
        self.layout: List[Tuple[str, int, Tuple[int, ...]]] = []
        name = C.create_string_buffer(128)
        off = C.c_longlong()
        shape = (C.c_int * 4)()
        nd = C.c_int()
        for i in range(self.lib.smd_num_tensors(h)):
            _lib.check(self.lib.smd_tensor_info(h, i, name, 128, C.byref(off), shape, C.byref(nd)))
            self.layout.append((name.value.decode(), int(off.value), tuple(shape[j] for j in range(nd.value))))
        self.arena_floats = int(self.lib.smd_arena_floats(h))
        self.workspace_bytes = int(self.lib.smd_workspace_bytes(h))
        self.device = device
        self._ws: Optional[torch.Tensor] = None
        self.params: Optional[torch.Tensor] = None
        self._sampler_T = 0

    def __del__(self):
        try:
            if getattr(self, "_plan", None):
                self.lib.smd_plan_destroy(self._plan)
                self._plan = None
        except Exception:
            pass

    # ------------------------------------------------------------------ parameter arena (host side)
    @property
    def num_params(self) -> int:
        return int(sum(int(np.prod(s)) for _, _, s in self.layout))

    def init_params(self, seed: int = 0, perturb: float = 0.0) -> np.ndarray:
        """flax.nn 0.3.0 default initialisers (Dense: lecun_normal kernel / zero bias; LayerNorm: ones / zeros).

        Same distributions as the reference, own RNG stream (seed-level init parity with flax is unpinned).
        ``perturb`` adds N(0, perturb) to every bias and LayerNorm parameter so tests exercise those paths.
        """
        rng = np.random.default_rng(seed)
        flat = np.zeros((self.arena_floats,), np.float32)
        for name, off, shape in self.layout:
            n = int(np.prod(shape))
            if name.endswith(".kernel"):
                fan_in = shape[0]
                std = np.sqrt(1.0 / fan_in) / 0.87962566103423978
                v = rng.standard_normal(n * 2)
                v = v[np.abs(v) <= 2.0][:n]
                while v.size < n:  # pragma: no cover
                    extra = rng.standard_normal(n)
                    v = np.concatenate([v, extra[np.abs(extra) <= 2.0]])[:n]
                val = (v * std).astype(np.float32)
            elif name.endswith(".scale"):
                val = np.ones((n,), np.float32)
            else:
                val = np.zeros((n,), np.float32)
            if perturb and not name.endswith(".kernel"):
                val = val + rng.normal(0.0, perturb, n).astype(np.float32)
            flat[off:off + n] = val
        return flat

    def flat_to_dict(self, flat) -> Dict[str, np.ndarray]:
        flat = flat.detach().cpu().numpy() if isinstance(flat, torch.Tensor) else np.asarray(flat)
        return {name: flat[off:off + int(np.prod(shape))].reshape(shape).copy() for name, off, shape in self.layout}

    def dict_to_flat(self, d: Dict[str, np.ndarray]) -> np.ndarray:
        flat = np.zeros((self.arena_floats,), np.float32)
        for name, off, shape in self.layout:
            flat[off:off + int(np.prod(shape))] = np.asarray(d[name], np.float32).reshape(-1)
        return flat

    # ------------------------------------------------------------------ device side
    def _stream(self) -> int:
        return torch.cuda.current_stream().cuda_stream

    def _ensure_ws(self) -> None:
        if self._ws is not None:
            return
        if not torch.cuda.is_available():
            raise _lib.SmdError("CUDA device required (libsmd has no CPU fallback)")
        dev = self.device or f"cuda:{torch.cuda.current_device()}"
        self._ws = torch.empty(self.workspace_bytes + 1024, dtype=torch.uint8, device=dev)
        base = self._ws.data_ptr()
        aligned = (base + 1023) // 1024 * 1024
        _lib.check(self.lib.smd_bind_workspace(self._plan, aligned, self.workspace_bytes))

    def set_params(self, flat) -> torch.Tensor:
        """Upload (or adopt) the fp32 arena and refresh the bf16 tensor-core operand copies."""
        self._ensure_ws()
        if isinstance(flat, np.ndarray):
            flat = torch.from_numpy(np.ascontiguousarray(flat, np.float32))
        if flat.numel() != self.arena_floats:
            raise ValueError("parameter arena has the wrong size")
        if not flat.is_cuda:
            flat = flat.to(self._ws.device)
        self.params = _f32c(flat, "params")
        self.repack()
        return self.params

    def repack(self) -> None:
        _lib.check(self.lib.smd_pack_weights(self._plan, self.params.data_ptr(), self._stream()))

    def forward(self, x: torch.Tensor, t: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """eps_hat = model(x, t); t has one value per example, or a single value (broadcast)."""
        x = _f32c(x, "x")
        batch = x.shape[0]
        t = _f32c(t.reshape(-1), "t")
        bcast = 1 if (t.numel() == 1 and batch > 1) else 0
        if not bcast and t.numel() != batch:
            raise ValueError("t must hold one value per example")
        y = torch.empty_like(x) if out is None else _f32c(out, "out")
        _lib.check(self.lib.smd_forward(self._plan, self.params.data_ptr(), x.data_ptr(), t.data_ptr(), bcast, batch,
                                        y.data_ptr(), self._stream()))
        return y

    def ddpm_loss(self, x0: torch.Tensor, used_alpha: torch.Tensor, eps: torch.Tensor, want_pred: bool = False):
        x0 = _f32c(x0, "x0"); eps = _f32c(eps, "eps"); ua = _f32c(used_alpha.reshape(-1), "used_alpha")
        batch = x0.shape[0]
        loss = torch.empty((batch,), dtype=torch.float32, device=x0.device)
        pred = torch.empty_like(x0) if want_pred else None
        _lib.check(self.lib.smd_ddpm_loss(self._plan, self.params.data_ptr(), x0.data_ptr(), ua.data_ptr(),
                                          eps.data_ptr(), batch, loss.data_ptr(), _ptr(pred), self._stream()))
        return (loss, pred) if want_pred else loss

    def ddpm_grads(self, x0, used_alpha, eps, grads: torch.Tensor, loss_sum: torch.Tensor, global_batch=None):
        x0 = _f32c(x0, "x0"); eps = _f32c(eps, "eps"); ua = _f32c(used_alpha.reshape(-1), "used_alpha")
        batch = x0.shape[0]
        _lib.check(self.lib.smd_ddpm_grads(self._plan, self.params.data_ptr(), x0.data_ptr(), ua.data_ptr(),
                                           eps.data_ptr(), batch, int(global_batch or batch), grads.data_ptr(),
                                           loss_sum.data_ptr(), self._stream()))

    def clip_adam(self, grads, m, v, lr: float, step: int, max_norm: float, scratch, gnorm, ema=None,
                  beta1=0.9, beta2=0.999, eps=1e-8, mu=0.999):
        _lib.check(self.lib.smd_clip_adam(self.params.data_ptr(), grads.data_ptr(), m.data_ptr(), v.data_ptr(),
                                          _ptr(ema), self.lib.smd_shadow_arena(self._plan), self.arena_floats, float(lr), int(step), float(max_norm),
                                          float(beta1), float(beta2), float(eps), float(mu), scratch.data_ptr(),
                                          gnorm.data_ptr(), self._stream()))

    # ------------------------------------------------------------------ objective draws (utils/losses.py:270-294)
    def objective_setup(self, betas: np.ndarray) -> None:
        self._ensure_ws()
        b = np.ascontiguousarray(betas, np.float32)
        _lib.check(self.lib.smd_objective_setup(self._plan, b.ctypes.data_as(C.POINTER(C.c_float)), len(b),
                                                self._stream()))

    def draws(self, key, batch: int, want_labels: bool = False, global_batch: Optional[int] = None,
              first_row: int = 0, continuous_noise: bool = True):
        """(used_alpha (B,), eps (B,S,C)[, labels]) from a jax PRNG key, generated on device.

        With ``global_batch`` / ``first_row`` the result is rows [first_row, first_row + batch) of the draws of a
        global batch (data-parallel ranks consume slices of ONE threefry stream: DP(seed) == single-GPU(seed))."""
        dev = self._ws.device
        shape = (batch, self.seq_len, self.cfg.channels) if ARCHS[self.cfg.arch] == 0 else (batch, self.cfg.channels)
        used = torch.empty((batch,), dtype=torch.float32, device=dev)
        eps = torch.empty(shape, dtype=torch.float32, device=dev)
        labels = torch.empty((batch,), dtype=torch.int32, device=dev) if want_labels else None
        k = (C.c_uint32 * 2)(int(key[0]) & 0xFFFFFFFF, int(key[1]) & 0xFFFFFFFF)
        _lib.check(self.lib.smd_ddpm_draws_sharded(self._plan, k, int(global_batch or batch), int(first_row), batch,
                                                   1 if continuous_noise else 0, used.data_ptr(), eps.data_ptr(),
                                                   _ptr(labels), self._stream()))
        return (used, eps, labels) if want_labels else (used, eps)

    # ------------------------------------------------------------------ NCSN family (SURVEY 8(f4))
    def dsm_setup(self, sigmas: np.ndarray) -> None:
        self._ensure_ws()
        s = np.ascontiguousarray(sigmas, np.float32)
        _lib.check(self.lib.smd_dsm_setup(self._plan, s.ctypes.data_as(C.POINTER(C.c_float)), len(s), self._stream()))

    def dsm_draws(self, key, batch: int, want_labels: bool = False, global_batch: Optional[int] = None,
                  first_row: int = 0, continuous_noise: bool = False):
        """(used_sigma (B,), eps[, labels]) of denoising_score_matching_loss (utils/losses.py:146-164) on device."""
        dev = self._ws.device
        shape = (batch, self.seq_len, self.cfg.channels) if ARCHS[self.cfg.arch] == 0 else (batch, self.cfg.channels)
        used = torch.empty((batch,), dtype=torch.float32, device=dev)
        eps = torch.empty(shape, dtype=torch.float32, device=dev)
        labels = torch.empty((batch,), dtype=torch.int32, device=dev) if want_labels else None
        k = (C.c_uint32 * 2)(int(key[0]) & 0xFFFFFFFF, int(key[1]) & 0xFFFFFFFF)
        _lib.check(self.lib.smd_dsm_draws(self._plan, k, int(global_batch or batch), int(first_row), batch,
                                          1 if continuous_noise else 0, used.data_ptr(), eps.data_ptr(), _ptr(labels),
                                          self._stream()))
        return (used, eps, labels) if want_labels else (used, eps)

    def dsm_loss(self, x0: torch.Tensor, used_sigma: torch.Tensor, eps: torch.Tensor, want_pred: bool = False):
        x0 = _f32c(x0, "x0"); eps = _f32c(eps, "eps"); us = _f32c(used_sigma.reshape(-1), "used_sigma")
        batch = x0.shape[0]
        loss = torch.empty((batch,), dtype=torch.float32, device=x0.device)
        pred = torch.empty_like(x0) if want_pred else None
        _lib.check(self.lib.smd_dsm_loss(self._plan, self.params.data_ptr(), x0.data_ptr(), us.data_ptr(), eps.data_ptr(),
                                         batch, loss.data_ptr(), _ptr(pred), self._stream()))
        return (loss, pred) if want_pred else loss

    def compute_dsm_grads(self, x0, used_sigma, eps, global_batch: Optional[int] = None) -> None:
        x0 = _f32c(x0, "x0"); eps = _f32c(eps, "eps"); us = _f32c(used_sigma.reshape(-1), "used_sigma")
        batch = x0.shape[0]
        _lib.check(self.lib.smd_dsm_grads(self._plan, self.params.data_ptr(), x0.data_ptr(), us.data_ptr(), eps.data_ptr(),
                                          batch, int(global_batch or batch), self.grads.data_ptr(),
                                          self._grads_buf[self.arena_floats:].data_ptr(), self._stream()))

    def ssm_draws(self, key, batch: int, want_labels: bool = False, global_batch: Optional[int] = None,
                  first_row: int = 0, continuous_noise: bool = False):
        """(used_sigma (B,), eps, v[, labels]) of sliced_score_matching_loss (utils/losses.py:203-223) on device; v holds
        the Rademacher (+-1) projection vectors.  Schedule: dsm_setup."""
        dev = self._ws.device
        shape = (batch, self.seq_len, self.cfg.channels) if ARCHS[self.cfg.arch] == 0 else (batch, self.cfg.channels)
        used = torch.empty((batch,), dtype=torch.float32, device=dev)
        eps = torch.empty(shape, dtype=torch.float32, device=dev)
        v = torch.empty(shape, dtype=torch.float32, device=dev)
        labels = torch.empty((batch,), dtype=torch.int32, device=dev) if want_labels else None
        k = (C.c_uint32 * 2)(int(key[0]) & 0xFFFFFFFF, int(key[1]) & 0xFFFFFFFF)
        _lib.check(self.lib.smd_ssm_draws(self._plan, k, int(global_batch or batch), int(first_row), batch,
                                          1 if continuous_noise else 0, used.data_ptr(), eps.data_ptr(), v.data_ptr(),
                                          _ptr(labels), self._stream()))
        return (used, eps, v, labels) if want_labels else (used, eps, v)

    def ssm_loss(self, x0: torch.Tensor, used_sigma: torch.Tensor, eps: torch.Tensor, v: torch.Tensor,
                 want_terms: bool = False):
        """Per-example sliced score matching loss; with want_terms also (score (B, C), v.J_s v (B,))."""
        x0 = _f32c(x0, "x0"); eps = _f32c(eps, "eps"); v = _f32c(v, "v")
        us = _f32c(used_sigma.reshape(-1), "used_sigma")
        batch = x0.shape[0]
        loss = torch.empty((batch,), dtype=torch.float32, device=x0.device)
        score = torch.empty_like(x0) if want_terms else None
        hvp = torch.empty((batch,), dtype=torch.float32, device=x0.device) if want_terms else None
        _lib.check(self.lib.smd_ssm_loss(self._plan, self.params.data_ptr(), x0.data_ptr(), us.data_ptr(), eps.data_ptr(),
                                         v.data_ptr(), batch, loss.data_ptr(), _ptr(score), _ptr(hvp), self._stream()))
        return (loss, score, hvp) if want_terms else loss

    def compute_ssm_grads(self, x0, used_sigma, eps, v, global_batch: Optional[int] = None) -> None:
        x0 = _f32c(x0, "x0"); eps = _f32c(eps, "eps"); v = _f32c(v, "v")
        us = _f32c(used_sigma.reshape(-1), "used_sigma")
        batch = x0.shape[0]
        _lib.check(self.lib.smd_ssm_grads(self._plan, self.params.data_ptr(), x0.data_ptr(), us.data_ptr(), eps.data_ptr(),
                                          v.data_ptr(), batch, int(global_batch or batch), self.grads.data_ptr(),
                                          self._grads_buf[self.arena_floats:].data_ptr(), self._stream()))

    def langevin_step(self, x, grad, alpha: float, noise_coef: float, step_key=None, z=None, infill_x=None,
                      infill_mask=None, infill_sigma: float = 0.0, infill_key=None, infill_z=None, x_next=None,
                      collection_slot=None, metrics4=None):
        x = _f32c(x, "x"); grad = _f32c(grad, "grad")
        x_next = torch.empty_like(x) if x_next is None else x_next
        mk = lambda k: None if k is None else (C.c_uint32 * 2)(int(k[0]) & 0xFFFFFFFF, int(k[1]) & 0xFFFFFFFF)
        _lib.check(self.lib.smd_langevin_step(self._plan, x.data_ptr(), grad.data_ptr(), x.shape[0], float(alpha),
                                              float(noise_coef), mk(step_key), _ptr(z), _ptr(infill_x), _ptr(infill_mask),
                                              float(infill_sigma), mk(infill_key), _ptr(infill_z), x_next.data_ptr(),
                                              _ptr(collection_slot), _ptr(metrics4), self._stream()))
        return x_next

    # ------------------------------------------------------------------ TransformerMDN (train_mdn.py)
    def _mdn_input(self, x: torch.Tensor) -> torch.Tensor:
        x = _f32c(x, "x")
        if x.dim() != 3 or tuple(x.shape[1:]) != (self.seq_len, self.cfg.channels):
            raise ValueError(f"x must have shape (batch, {self.seq_len}, {self.cfg.channels}), got {tuple(x.shape)}")
        return x

    def mdn_forward(self, x: torch.Tensor, shift: bool = True):
        """(pi (B,S,Kc), mu (B,S,Kc*C), log_sigma (B,S,Kc*C)) = model(x, shift) (models/autoregressive.py:40-82)."""
        x = self._mdn_input(x)
        B, S, Cc = x.shape
        kc = self.cfg.mdn_components
        pi = torch.empty((B, S, kc), dtype=torch.float32, device=x.device)
        mu = torch.empty((B, S, kc * Cc), dtype=torch.float32, device=x.device)
        ls = torch.empty_like(mu)
        _lib.check(self.lib.smd_mdn_forward(self._plan, self.params.data_ptr(), x.data_ptr(), B, 1 if shift else 0,
                                            pi.data_ptr(), mu.data_ptr(), ls.data_ptr(), self._stream()))
        return pi, mu, ls

    def mdn_loss(self, x: torch.Tensor) -> torch.Tensor:
        """Per-token negative log-likelihood (B*S,) of eval_step (train_mdn.py:154-168)."""
        x = self._mdn_input(x)
        loss = torch.empty((x.shape[0] * x.shape[1],), dtype=torch.float32, device=x.device)
        _lib.check(self.lib.smd_mdn_loss(self._plan, self.params.data_ptr(), x.data_ptr(), x.shape[0], loss.data_ptr(),
                                         self._stream()))
        return loss

    def compute_mdn_grads(self, x: torch.Tensor, global_batch: Optional[int] = None) -> None:
        """grads <- d(mean token NLL over the GLOBAL batch)/d params for this shard; loss_sum / loss_mean as
        compute_grads (loss_mean: the token mean)."""
        x = self._mdn_input(x)
        _lib.check(self.lib.smd_mdn_grads(self._plan, self.params.data_ptr(), x.data_ptr(), x.shape[0],
                                          int(global_batch or x.shape[0]), self.grads.data_ptr(),
                                          self._grads_buf[self.arena_floats:].data_ptr(), self._stream()))

    # ------------------------------------------------------------------ optimizer step (train_ncsn.py:260-288)
    def init_train_state(self, ema: bool = False) -> None:
        """Allocates gradient / Adam moment (/ EMA) arenas next to the parameter arena (flax.optim.Adam state)."""
        if not self.training:
            raise _lib.SmdError("Engine was created with training=False")
        if self.params is None:
            raise _lib.SmdError("set_params() first")
        dev = self.params.device
        n = self.arena_floats
        # the loss accumulator sits right behind the gradient arena so that one collective reduces both
        self._grads_buf = torch.zeros(n + 8, dtype=torch.float32, device=dev)
        self.grads = self._grads_buf[:n]
        self.adam_m = torch.zeros(n, dtype=torch.float32, device=dev)
        self.adam_v = torch.zeros(n, dtype=torch.float32, device=dev)
        self.ema_params = self.params.clone() if ema else None
        self._scratch = torch.zeros(1024, dtype=torch.float32, device=dev)
        self.grad_norm = torch.zeros(1, dtype=torch.float32, device=dev)
        self.loss_sum = self._grads_buf[n:n + 1]       # sum of this shard's per-example losses
        self.loss_mean = self._grads_buf[n + 1:n + 2]  # loss_sum / global batch (SUM over ranks = global mean loss)
        self.opt_step = 0

    def compute_grads(self, x0, used_alpha, eps, global_batch: Optional[int] = None) -> None:
        """grads <- d(mean over the GLOBAL batch of the loss)/d params for this shard; loss_sum <- sum of losses."""
        self.ddpm_grads(x0, used_alpha, eps, self.grads, self._grads_buf[self.arena_floats:], global_batch)

    def reduce_grads(self, world_size: int, process_group=None) -> None:
        """SUM all-reduce of the gradient arena and the loss scalar over the data-parallel ranks (call right after
        compute_grads; the current stream ends up waiting for the reduced gradients)."""
        if world_size <= 1:
            return
        import torch.distributed as dist
        overlap = self.grads.is_cuda and dist.get_backend(process_group) == "nccl" and \
            os.environ.get("SMD_DP_OVERLAP", "1") != "0"
        if overlap:
            # the tail / output-layer gradients (~85% of the arena) are final before the trunk backward starts:
            # their all-reduce runs on a communication stream underneath it (include/smd.h: smd_wait_tail_grads)
            first, count = self.grads_tail_range()
            if self._comm_stream is None:
                self._comm_stream = torch.cuda.Stream()
            with torch.cuda.stream(self._comm_stream):
                _lib.check(self.lib.smd_wait_tail_grads(self._plan, C.c_void_p(self._comm_stream.cuda_stream)))
                # + 2: the loss scalars stored behind the arena ride along (final long before the tail gradients)
                w_tail = dist.all_reduce(self._grads_buf[first:first + count + 2], op=dist.ReduceOp.SUM,
                                         group=process_group, async_op=True)
            w_head = dist.all_reduce(self.grads[:first], op=dist.ReduceOp.SUM, group=process_group, async_op=True)
            w_head.wait()
            w_tail.wait()      # the current stream now waits for both reductions
        else:
            dist.all_reduce(self._grads_buf[:self.grads.numel() + 2], op=dist.ReduceOp.SUM, group=process_group)

    def grads_tail_range(self):
        """(first_float, num_floats) of the gradient-arena slice that is final after the tail backward."""
        first, count = C.c_longlong(0), C.c_longlong(0)
        _lib.check(self.lib.smd_grads_tail_range(self._plan, C.byref(first), C.byref(count)))
        return int(first.value), int(count.value)

    def apply_grads(self, lr: float, grad_clip: float = 1.0, mu: float = 0.999) -> None:
        self.clip_adam(self.grads, self.adam_m, self.adam_v, lr, self.opt_step, grad_clip, self._scratch,
                       self.grad_norm, ema=self.ema_params, mu=mu)
        self.opt_step += 1
        # the fused clip+Adam kernel already refreshed the bf16 shadow arena; only the padded out.kernel copy is left
        _lib.check(self.lib.smd_pack_weights_after_adam(self._plan, self.params.data_ptr(), self._stream()))

    def train_step(self, x0, used_alpha, eps, lr: float, grad_clip: float = 1.0, process_group=None,
                   world_size: int = 1):
        """One data-parallel optimizer step: local grads -> NCCL all-reduce(sum) -> clip -> Adam.

        Returns (mean loss over the global batch, post-clip grad norm) as device tensors (no host sync)."""
        batch = x0.shape[0]
        self.compute_grads(x0, used_alpha, eps, global_batch=batch * world_size)
        self.reduce_grads(world_size, process_group)
        self.apply_grads(lr, grad_clip)
        return self.loss_mean, self.grad_norm

    # ------------------------------------------------------------------ sampler
    def sampler_setup(self, betas: np.ndarray, key=(0, 0)) -> None:
        self._ensure_ws()
        b = np.ascontiguousarray(betas, np.float32)
        k = (C.c_uint32 * 2)(int(key[0]) & 0xFFFFFFFF, int(key[1]) & 0xFFFFFFFF)
        _lib.check(self.lib.smd_sampler_setup(self._plan, b.ctypes.data_as(C.POINTER(C.c_float)), len(b), k,
                                              self._stream()))
        self._sampler_T = len(b)

    def set_sampler_shard(self, first_row: int = 0, total_rows: int = 0) -> None:
        """This engine's sampler calls hold samples [first_row, ...) of a global batch of total_rows samples and draw
        that slice of the chain's threefry streams (0, 0: off)."""
        _lib.check(self.lib.smd_sampler_set_shard(self._plan, int(first_row), int(total_rows)))

    def reverse_step(self, x, t: int, z=None, infill_x=None, infill_mask=None, infill_z=None, x_next=None,
                     eps_hat=None, collection=None, metrics=None):
        x = _f32c(x, "x")
        x_next = torch.empty_like(x) if x_next is None else x_next
        _lib.check(self.lib.smd_ddpm_reverse_step(self._plan, self.params.data_ptr(), x.data_ptr(), x.shape[0],
                                                  int(t), _ptr(z), _ptr(infill_x), _ptr(infill_mask), _ptr(infill_z),
                                                  x_next.data_ptr(), _ptr(eps_hat), _ptr(collection), _ptr(metrics),
                                                  self._stream()))
        return x_next

    def sample(self, x, steps: Optional[int] = None, infill_x=None, infill_mask=None, collection=None,
               metrics=None, use_graph: bool = True):
        """Runs `steps` reverse steps in place on x (n, S, C)."""
        x = _f32c(x, "x")
        steps = self._sampler_T if steps is None else int(steps)
        _lib.check(self.lib.smd_ddpm_sample(self._plan, self.params.data_ptr(), x.data_ptr(), x.shape[0], steps,
                                            _ptr(infill_x), _ptr(infill_mask), _ptr(collection), _ptr(metrics),
                                            1 if use_graph else 0, self._stream()))
        return x

    def launch_count(self) -> int:
        return int(self.lib.smd_launch_count())

    def describe(self) -> dict:
        d = asdict(self.cfg)
        d.update(params=self.num_params, arena_floats=self.arena_floats, workspace_mb=self.workspace_bytes / 2 ** 20)
        return d
