"""Checkpoint save / restore with the call shape of flax.training.checkpoints (train_ncsn.py:395-399,
sample_ncsn.py:341-342): save_checkpoint(dir, (optimizer, ema, early_stop), step, keep=N) writes
``checkpoint_<step>`` atomically and prunes to the newest `keep`; restore_checkpoint(dir, target) loads the
latest into the template objects.  train_mdn.py:305-307 saves the 2-tuple (optimizer, early_stop) instead: its
state dict is {'0': optimizer, '1': early_stop}, as flax's to_state_dict writes any tuple.

Default format: msgpack of a state dict {'0': optimizer, '1': ema, '2': early_stop} with the flat arenas as ndarray
leaves encoded as {'__nd__': True, 'dtype', 'shape', 'data'} plus the arena layout (self-describing).
With SMD_CHECKPOINT_FORMAT=flax (or save_checkpoint(..., fmt="flax")) the file is written in flax 0.3.0's own wire
format -- nested pre-Linen parameter tree, msgpack ext-type ndarrays (flax_compat.py; restated from memory, not
verifiable here); restore_checkpoint detects either format."""
from __future__ import annotations

import os
import re

import msgpack
import numpy as np
import torch

PREFIX = "checkpoint_"


def _nd(a) -> dict:
    a = np.ascontiguousarray(a)
    return {"__nd__": True, "dtype": str(a.dtype), "shape": list(a.shape), "data": a.tobytes()}


def _un_nd(d) -> np.ndarray:
    return np.frombuffer(d["data"], dtype=np.dtype(d["dtype"])).reshape(d["shape"]).copy()


def split_target(target):
    """(optimizer, ema, early_stop) or train_mdn's (optimizer, early_stop) -> (optimizer, ema or None, early_stop)"""
    if len(target) == 2:
        return target[0], None, target[1]
    return tuple(target)


def join_target(target, optimizer, ema, early_stop):
    return (optimizer, early_stop) if len(target) == 2 else (optimizer, ema, early_stop)


def _state(target) -> dict:
    optimizer, ema, early_stop = split_target(target)
    opt = {"state": {"step": int(optimizer.step), "grad_ema": _nd(optimizer.grad_ema.cpu().numpy()),
                     "grad_sq_ema": _nd(optimizer.grad_sq_ema.cpu().numpy())},
           "target": {"params": _nd(optimizer.target.arena.flat.cpu().numpy()),
                      "layout": [[n, int(o), list(s)] for n, o, s in optimizer.target.arena.layout]}}
    if len(target) == 2:
        return {"0": opt, "1": early_stop.state_dict()}
    e = None if ema is None else {"mu": float(ema.mu), "params": _nd(ema.params.flat.cpu().numpy())}
    return {"0": opt, "1": e, "2": early_stop.state_dict()}


def _natural_key(name: str):
    return [int(t) if t.isdigit() else t for t in re.split(r"(\d+)", name)]


def list_checkpoints(ckpt_dir: str, prefix: str = PREFIX):
    if not os.path.isdir(ckpt_dir):
        return []
    names = [n for n in os.listdir(ckpt_dir) if n.startswith(prefix) and not n.endswith(".tmp")]
    return sorted(names, key=_natural_key)


def save_checkpoint(ckpt_dir: str, target, step: int, prefix: str = PREFIX, keep: int = 1, fmt: str = None) -> str:
    os.makedirs(ckpt_dir, exist_ok=True)
    path = os.path.join(ckpt_dir, f"{prefix}{step}")
    tmp = path + ".tmp"
    fmt = fmt or os.environ.get("SMD_CHECKPOINT_FORMAT", "native")
    if fmt not in ("native", "flax"):
        raise ValueError(f"unknown checkpoint format {fmt!r}")
    if fmt == "flax":
        from . import flax_compat
        blob = flax_compat.msgpack_serialize(flax_compat.to_flax_state(target))
    else:
        blob = msgpack.packb(_state(target), use_bin_type=True)
    with open(tmp, "wb") as f:
        f.write(blob)
    os.replace(tmp, path)
    names = list_checkpoints(ckpt_dir, prefix)
    for old in names[:-keep] if keep > 0 else []:
        os.remove(os.path.join(ckpt_dir, old))
    return path


def restore_checkpoint(ckpt_dir: str, target, step: int = None, prefix: str = PREFIX):
    """Loads the newest (or the given) checkpoint INTO the template objects and returns them; returns the template
    untouched when the directory holds no checkpoint (flax behaviour)."""
    names = list_checkpoints(ckpt_dir, prefix)
    if step is not None:
        names = [n for n in names if n == f"{prefix}{step}"]
    if not names:
        return target
    from . import flax_compat
    with open(os.path.join(ckpt_dir, names[-1]), "rb") as f:
        st = flax_compat.msgpack_restore(f.read())       # plain msgpack plus flax's ndarray ext types
    if flax_compat.is_flax_state(st):
        return flax_compat.load_flax_state(st, target)
    optimizer, ema, early_stop = split_target(target)
    o = st["0"]
    flat = _un_nd(o["target"]["params"])
    arena = optimizer.target.arena
    if flat.size != arena.flat.numel():
        raise ValueError("checkpoint parameter arena does not match the model (different flags?)")
    arena.flat.copy_(torch.from_numpy(flat))
    arena.bump()
    optimizer.step = int(o["state"]["step"])
    optimizer.grad_ema.copy_(torch.from_numpy(_un_nd(o["state"]["grad_ema"])))
    optimizer.grad_sq_ema.copy_(torch.from_numpy(_un_nd(o["state"]["grad_sq_ema"])))
    if ema is not None and st.get("1") is not None:
        ema.params.flat.copy_(torch.from_numpy(_un_nd(st["1"]["params"])))
        ema.params.bump()
        ema.mu = float(st["1"]["mu"])
    from .train_utils import EarlyStopping
    es_key = "1" if len(target) == 2 else "2"
    es = EarlyStopping(**st[es_key]) if st.get(es_key) else early_stop
    return join_target(target, optimizer, ema, es)
