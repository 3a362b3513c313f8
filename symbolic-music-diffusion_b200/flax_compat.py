"""flax-0.3.0 checkpoint wire format for `(optimizer, ema, early_stop)` (SURVEY section 8, row f1), and for the
`(optimizer, early_stop)` 2-tuple of train_mdn.py:305-307 ({'0': optimizer, '1': early_stop}).  TransformerMDN's
parameter tree (models/autoregressive.py:49-82): the TransformerDDPM trunk indices, DenseResBlock_{4+5L+k},
LayerNorm_{4+5L+K} and the explicitly named `mdn` module with Dense_0 / Dense_1 / Dense_2 = mu / log_sigma / pi
(models/shared.py MDN) -- restated like the rest of this module, not verified against flax.

What the reference writes (train_ncsn.py:395-399 -> flax.training.checkpoints.save_checkpoint ->
flax.serialization.to_bytes): msgpack of `to_state_dict(target)` where
  * a tuple becomes {'0': ..., '1': ..., '2': ...};
  * flax.optim.Optimizer -> {'state': {'step': int32 scalar, 'param_states': <params tree of
    {'grad_ema', 'grad_sq_ema'}>}, 'target': {'params': <params tree>}}   (flax.optim.Adam, pre-Linen nn.Model);
  * EMAHelper -> {'mu', 'params'},  EarlyStopping -> its five fields  (utils/train_utils.py:25-78);
  * every ndarray leaf is msgpack ExtType(1, packb((shape, dtype.name, C-order bytes))), numpy scalars ExtType(3, same).

The parameter tree uses pre-Linen flax.nn auto-names `ClassName_<i>`, `i` counting ALL submodules created so far in
the parent (also the parameter-less ones: TransformerPositionalEncoding, NoiseEncoding, FeaturewiseAffine), and the
explicit names query / key / value / out inside the attention block, which is auto-named after its base class
`MultiHeadDotProductAttention_<i>` (nn.SelfAttention is a .partial of it)  (models/ncsn.py:122-179,
models/shared.py:33-75).

NOT VERIFIED against flax itself: neither flax 0.3.0 nor a checkpoint written by it can exist in this environment.
Both conventions above are restated from the flax 0.3.0 sources as remembered; `tests/test_flax_compat.py` pins the
byte layout of the encoder and the round trip, not agreement with flax.  The repository's own default checkpoint
format stays the self-describing one in checkpoints.py; this module is opt-in (`SMD_CHECKPOINT_FORMAT=flax`,
restore auto-detects)."""
from __future__ import annotations

from typing import Dict, Tuple

import msgpack
import numpy as np

_EXT_NDARRAY, _EXT_NPSCALAR = 1, 3


# ------------------------------------------------------------------------------------------------ msgpack leaves
def _nd_bytes(a: np.ndarray) -> bytes:
    a = np.asarray(a)
    return msgpack.packb((list(a.shape), a.dtype.name, a.tobytes("C")), use_bin_type=True)


def _ext_pack(x):
    if isinstance(x, np.ndarray):
        return msgpack.ExtType(_EXT_NDARRAY, _nd_bytes(x))
    if isinstance(x, np.generic):
        return msgpack.ExtType(_EXT_NPSCALAR, _nd_bytes(np.asarray(x)))
    raise TypeError(f"cannot serialise {type(x)}")


def _ext_unpack(code, data):
    if code in (_EXT_NDARRAY, _EXT_NPSCALAR):
        shape, dtype_name, buf = msgpack.unpackb(data, raw=True)
        name = dtype_name.decode() if isinstance(dtype_name, bytes) else dtype_name
        arr = np.frombuffer(buf, dtype=np.dtype(name)).reshape(shape)
        return arr[()] if code == _EXT_NPSCALAR else arr.copy()
    return msgpack.ExtType(code, data)


def msgpack_serialize(tree) -> bytes:
    return msgpack.packb(tree, default=_ext_pack, strict_types=True, use_bin_type=True)


def msgpack_restore(data: bytes):
    return msgpack.unpackb(data, ext_hook=_ext_unpack, raw=False, strict_map_key=False)


# ------------------------------------------------------------------------------------------------ parameter tree
def _tree_paths(cfg) -> Dict[str, Tuple[Tuple[str, ...], str]]:
    """arena tensor name -> (flax path of the module, kind); kind selects how the leaf / leaves are laid out."""
    out: Dict[str, Tuple[Tuple[str, ...], str]] = {}

    def film_res(prefix_k: str, film: str, res: str):
        out[f"{prefix_k}.film.d1"] = ((film, "Dense_1"), "dense")
        out[f"{prefix_k}.film.d2"] = ((film, "Dense_2"), "dense")
        out[f"{prefix_k}.film.ss"] = ((film,), "scale_shift")          # Dense_3 (scale) | Dense_4 (shift)
        out[f"{prefix_k}.res.ln_a"] = ((res, "LayerNorm_0"), "ln")
        out[f"{prefix_k}.res.a"] = ((res, "Dense_2"), "dense")
        out[f"{prefix_k}.res.ln_b"] = ((res, "LayerNorm_3"), "ln")
        out[f"{prefix_k}.res.b"] = ((res, "Dense_5"), "dense")

    if cfg.arch == "DenseDDPM":
        n = cfg.num_layers
        out["in"] = (("Dense_0",), "dense")
        for i in range(n):
            film_res(f"k{i}", f"DenseFiLM_{1 + 2 * i}", f"DenseResBlock_{2 + 2 * i}")
        out["out_ln"] = ((f"LayerNorm_{1 + 2 * n}",), "ln")
        out["out"] = ((f"Dense_{2 + 2 * n}",), "dense")
        return out
    L, K = cfg.num_layers, cfg.num_mlp_layers
    mdn = cfg.arch == "TransformerMDN"
    out["in"] = (("Dense_1",), "dense")                                  # index 0 is TransformerPositionalEncoding
    for l in range(L):
        b = 2 + 5 * l
        out[f"l{l}.ln1"] = ((f"LayerNorm_{b}",), "ln")
        # nn.SelfAttention is MultiHeadDotProductAttention.partial(inputs_kv=None); pre-Linen Module.partial keeps the
        # base class __name__, so the auto-name is MultiHeadDotProductAttention_<i> (as in pre-Linen ViT checkpoints).
        # `SelfAttention_<i>` (what round 1 wrote) is still accepted on restore (_ALIASES).
        out[f"l{l}.attn.qkv"] = ((f"MultiHeadDotProductAttention_{b + 1}",), "qkv")
        out[f"l{l}.attn.out"] = ((f"MultiHeadDotProductAttention_{b + 1}", "out"), "attn_out")
        out[f"l{l}.ln2"] = ((f"LayerNorm_{b + 2}",), "ln")
        out[f"l{l}.ffn1"] = ((f"Dense_{b + 3}",), "dense")
        out[f"l{l}.ffn2"] = ((f"Dense_{b + 4}",), "dense")
    b = 2 + 5 * L
    out["post_ln"] = ((f"LayerNorm_{b}",), "ln")
    out["post"] = ((f"Dense_{b + 1}",), "dense")
    if mdn:   # DenseResBlock(x, mlp_dims) without a FiLM generator: one submodule per block
        for k in range(K):
            res = f"DenseResBlock_{b + 2 + k}"
            out[f"k{k}.res.ln_a"] = ((res, "LayerNorm_0"), "ln")
            out[f"k{k}.res.a"] = ((res, "Dense_2"), "dense")
            out[f"k{k}.res.ln_b"] = ((res, "LayerNorm_3"), "ln")
            out[f"k{k}.res.b"] = ((res, "Dense_5"), "dense")
        out["out_ln"] = ((f"LayerNorm_{b + 2 + K}",), "ln")
        out["mdn.mu"] = (("mdn", "Dense_0"), "dense")
        out["mdn.log_sigma"] = (("mdn", "Dense_1"), "dense")
        out["mdn.pi"] = (("mdn", "Dense_2"), "dense")
        return out
    for k in range(K):
        film_res(f"k{k}", f"DenseFiLM_{b + 2 + 2 * k}", f"DenseResBlock_{b + 3 + 2 * k}")
    out["out_ln"] = ((f"LayerNorm_{b + 2 + 2 * K}",), "ln")
    out["out"] = ((f"Dense_{b + 3 + 2 * K}",), "dense")
    return out


def _node(tree: dict, path) -> dict:
    for p in path:
        tree = tree.setdefault(p, {})
    return tree


def params_to_flax(arena: Dict[str, np.ndarray], cfg) -> dict:
    """{arena tensor name: ndarray} -> the nested parameter dict flax.nn would hold for this model."""
    H = getattr(cfg, "num_heads", 8)
    tree: dict = {}
    for mod, (path, kind) in _tree_paths(cfg).items():
        if kind == "ln":
            _node(tree, path).update(scale=np.asarray(arena[mod + ".scale"]), bias=np.asarray(arena[mod + ".bias"]))
        elif kind == "dense":
            _node(tree, path).update(kernel=np.asarray(arena[mod + ".kernel"]), bias=np.asarray(arena[mod + ".bias"]))
        elif kind == "scale_shift":
            w, b = np.asarray(arena[mod + ".kernel"]), np.asarray(arena[mod + ".bias"])
            m = w.shape[1] // 2
            _node(tree, path + ("Dense_3",)).update(kernel=w[:, :m].copy(), bias=b[:m].copy())
            _node(tree, path + ("Dense_4",)).update(kernel=w[:, m:].copy(), bias=b[m:].copy())
        elif kind == "qkv":
            w, b = np.asarray(arena[mod + ".kernel"]), np.asarray(arena[mod + ".bias"])
            e = w.shape[0]
            for i, name in enumerate(("query", "key", "value")):
                _node(tree, path + (name,)).update(kernel=w[:, i * e:(i + 1) * e].reshape(e, H, e // H).copy(),
                                                   bias=b[i * e:(i + 1) * e].reshape(H, e // H).copy())
        elif kind == "attn_out":
            w = np.asarray(arena[mod + ".kernel"])
            _node(tree, path).update(kernel=w.reshape(H, w.shape[0] // H, w.shape[1]).copy(),
                                     bias=np.asarray(arena[mod + ".bias"]))
    return tree


def params_from_flax(tree: dict, cfg) -> Dict[str, np.ndarray]:
    """Inverse of params_to_flax; parameter-less submodules (possibly present as empty dicts) are ignored."""
    out: Dict[str, np.ndarray] = {}

    def get(path):
        node = tree
        for p in path:
            if p not in node:
                alt = p.replace("MultiHeadDotProductAttention_", "SelfAttention_")
                if alt not in node:
                    raise KeyError("flax parameter tree has no " + "/".join(path))
                p = alt
            node = node[p]
        return node

    for mod, (path, kind) in _tree_paths(cfg).items():
        if kind == "ln":
            n = get(path)
            out[mod + ".scale"], out[mod + ".bias"] = np.asarray(n["scale"]), np.asarray(n["bias"])
        elif kind == "dense":
            n = get(path)
            out[mod + ".kernel"], out[mod + ".bias"] = np.asarray(n["kernel"]), np.asarray(n["bias"])
        elif kind == "scale_shift":
            s, h = get(path + ("Dense_3",)), get(path + ("Dense_4",))
            out[mod + ".kernel"] = np.concatenate([np.asarray(s["kernel"]), np.asarray(h["kernel"])], axis=1)
            out[mod + ".bias"] = np.concatenate([np.asarray(s["bias"]), np.asarray(h["bias"])], axis=0)
        elif kind == "qkv":
            ws, bs = [], []
            for name in ("query", "key", "value"):
                n = get(path + (name,))
                w = np.asarray(n["kernel"])
                ws.append(w.reshape(w.shape[0], -1))
                bs.append(np.asarray(n["bias"]).reshape(-1))
            out[mod + ".kernel"], out[mod + ".bias"] = np.concatenate(ws, axis=1), np.concatenate(bs, axis=0)
        elif kind == "attn_out":
            n = get(path)
            w = np.asarray(n["kernel"])
            out[mod + ".kernel"], out[mod + ".bias"] = w.reshape(-1, w.shape[-1]), np.asarray(n["bias"])
    return out


# ------------------------------------------------------------------------------------------------ whole target
def _flat_to_named(flat: np.ndarray, layout) -> Dict[str, np.ndarray]:
    return {n: flat[o:o + int(np.prod(s))].reshape(s) for n, o, s in layout}


def _named_to_flat(named: Dict[str, np.ndarray], layout, size: int) -> np.ndarray:
    flat = np.zeros(size, np.float32)
    for n, o, s in layout:
        a = np.asarray(named[n], np.float32)
        if tuple(a.shape) != tuple(s):
            raise ValueError(f"{n}: checkpoint shape {a.shape} != model shape {tuple(s)}")
        flat[o:o + a.size] = a.reshape(-1)
    return flat


def to_flax_state(target) -> dict:
    """State dict of (optimizer, ema, early_stop) -- or (optimizer, early_stop) -- in flax's layout (numpy leaves)."""
    from .checkpoints import split_target
    optimizer, ema, early_stop = split_target(target)
    arena = optimizer.target.arena
    cfg = arena.spec.model_config(arena.input_shape)
    layout = arena.layout
    npf = lambda t: t.detach().cpu().numpy()
    params = params_to_flax(_flat_to_named(npf(arena.flat), layout), cfg)
    gm = params_to_flax(_flat_to_named(npf(optimizer.grad_ema), layout), cfg)
    gv = params_to_flax(_flat_to_named(npf(optimizer.grad_sq_ema), layout), cfg)

    def zip_states(a, b):
        if isinstance(a, dict):
            return {k: zip_states(a[k], b[k]) for k in a}
        return {"grad_ema": a, "grad_sq_ema": b}

    opt = {"state": {"step": np.asarray(int(optimizer.step), np.int32), "param_states": zip_states(gm, gv)},
           "target": {"params": params}}
    e = None
    if ema is not None:
        e = {"mu": float(ema.mu), "params": params_to_flax(_flat_to_named(npf(ema.params.flat), layout), cfg)}
    es = early_stop.state_dict()
    if len(target) == 2:
        return {"0": opt, "1": es}
    return {"0": opt, "1": e, "2": es}


def is_flax_state(st) -> bool:
    try:
        return "param_states" in st["0"]["state"]
    except (KeyError, TypeError):
        return False


def load_flax_state(st: dict, target):
    """Fill the template objects from a flax-layout state dict (inverse of to_flax_state)."""
    import torch
    from .checkpoints import join_target, split_target
    from .train_utils import EarlyStopping
    optimizer, ema, early_stop = split_target(target)
    arena = optimizer.target.arena
    cfg = arena.spec.model_config(arena.input_shape)
    layout, size = arena.layout, arena.flat.numel()

    def unzip(tree, key):
        if isinstance(tree, dict) and "grad_ema" in tree and "grad_sq_ema" in tree and not isinstance(tree["grad_ema"], dict):
            return tree[key]
        return {k: unzip(v, key) for k, v in tree.items()}

    o = st["0"]
    put = lambda dst, tree: dst.copy_(torch.from_numpy(_named_to_flat(params_from_flax(tree, cfg), layout, size)))
    put(arena.flat, o["target"]["params"])
    arena.bump()
    optimizer.step = int(np.asarray(o["state"]["step"]))
    put(optimizer.grad_ema, unzip(o["state"]["param_states"], "grad_ema"))
    put(optimizer.grad_sq_ema, unzip(o["state"]["param_states"], "grad_sq_ema"))
    if ema is not None and st.get("1") is not None:
        put(ema.params.flat, st["1"]["params"])
        ema.params.bump()
        ema.mu = float(np.asarray(st["1"]["mu"]))
    es = early_stop
    es_key = "1" if len(target) == 2 else "2"
    if st.get(es_key):
        d = {k: (v.item() if isinstance(v, np.generic) else v) for k, v in st[es_key].items()}
        es = EarlyStopping(**d)
    return join_target(target, optimizer, ema, es)
