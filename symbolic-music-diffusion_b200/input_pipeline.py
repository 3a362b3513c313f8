"""TensorFlow-free input pipeline with the reference's behaviour (input_pipeline.py:113-235, utils/data_utils.py):

TFRecord shards ``{dataset}/{train,eval}-*.tfrecord`` of ``tf.train.Example{inputs: FloatList, input_shape:
Int64List}`` (written by scripts/transform_encoded_data.py:71-92) -> shuffle buffer 8 x batch -> batch with
drop_remainder -> optional dim-weights multiply and slice gather (input_pipeline.py:43-48) -> one global scalar
min / max per split, cached as ``{dataset}/cache/{split}_{config}_{min,max}.pkl`` -> normalise to [-1, 1]
(input_pipeline.py:36-40).  ``ds.examples`` is the number of BATCHES per epoch (data_utils.py:63-90), cached as
``cache/{split}_{batch}_cardinality.pkl``.  PCA checkpoints need scikit-learn pickles and are honoured if given.
"""
from __future__ import annotations

import glob
import os
import pickle
import struct
from typing import Iterator, List, Optional, Sequence

import numpy as np

# ------------------------------------------------------------------------------------------------ crc32c / TFRecord
_CRC_TABLE: Optional[np.ndarray] = None


def _crc_table() -> np.ndarray:
    global _CRC_TABLE
    if _CRC_TABLE is None:
        tab = np.zeros(256, dtype=np.uint32)
        for i in range(256):
            c = i
            for _ in range(8):
                c = (c >> 1) ^ 0x82F63B78 if c & 1 else c >> 1
            tab[i] = c
        _CRC_TABLE = tab
    return _CRC_TABLE


def crc32c(data: bytes) -> int:
    tab = _crc_table()
    c = 0xFFFFFFFF
    for b in data:
        c = int(tab[(c ^ b) & 0xFF]) ^ (c >> 8)
    return c ^ 0xFFFFFFFF


def masked_crc(data: bytes) -> int:
    c = crc32c(data)
    return ((((c >> 15) | (c << 17)) & 0xFFFFFFFF) + 0xA282EAD8) & 0xFFFFFFFF


def read_tfrecord(path: str, verify: bool = False) -> Iterator[bytes]:
    """Yields the payload of every record: [u64 len][u32 masked crc(len)][payload][u32 masked crc(payload)]."""
    with open(path, "rb") as f:
        while True:
            head = f.read(12)
            if not head:
                return
            if len(head) < 12:
                raise ValueError(f"{path}: truncated TFRecord header")
            (n,) = struct.unpack("<Q", head[:8])
            if verify and struct.unpack("<I", head[8:])[0] != masked_crc(head[:8]):
                raise ValueError(f"{path}: corrupt TFRecord length CRC")
            payload = f.read(n)
            tail = f.read(4)
            if len(payload) < n or len(tail) < 4:
                raise ValueError(f"{path}: truncated TFRecord payload")
            if verify and struct.unpack("<I", tail)[0] != masked_crc(payload):
                raise ValueError(f"{path}: corrupt TFRecord payload CRC")
            yield payload


def write_tfrecord(path: str, payloads: Sequence[bytes]) -> None:
    with open(path, "wb") as f:
        for p in payloads:
            head = struct.pack("<Q", len(p))
            f.write(head + struct.pack("<I", masked_crc(head)) + p + struct.pack("<I", masked_crc(p)))


# ------------------------------------------------------------------------------------------------ tf.train.Example
def _varint(buf: bytes, pos: int):
    out, shift = 0, 0
    while True:
        b = buf[pos]
        pos += 1
        out |= (b & 0x7F) << shift
        if not b & 0x80:
            return out, pos
        shift += 7


def _fields(buf: bytes):
    """(field number, wire type, value) triples of one protobuf message."""
    pos, n = 0, len(buf)
    while pos < n:
        key, pos = _varint(buf, pos)
        num, wt = key >> 3, key & 7
        if wt == 0:
            v, pos = _varint(buf, pos)
        elif wt == 1:
            v = buf[pos:pos + 8]; pos += 8
        elif wt == 2:
            ln, pos = _varint(buf, pos)
            v = buf[pos:pos + ln]; pos += ln
        elif wt == 5:
            v = buf[pos:pos + 4]; pos += 4
        else:
            raise ValueError(f"unsupported protobuf wire type {wt}")
        yield num, wt, v


def parse_example(payload: bytes) -> dict:
    """Minimal tf.train.Example parser: {feature name: np.ndarray (float32 / int64) or list of bytes}."""
    out = {}
    for num, _, features in _fields(payload):
        if num != 1:
            continue
        for fnum, _, entry in _fields(features):          # map<string, Feature> entries
            if fnum != 1:
                continue
            name, feat = None, b""
            for enum, _, v in _fields(entry):
                if enum == 1:
                    name = v.decode("utf-8")
                elif enum == 2:
                    feat = v
            for kind, _, lst in _fields(feat):             # oneof bytes_list=1 / float_list=2 / int64_list=3
                if kind == 2:
                    vals: List[np.ndarray] = []
                    for vnum, wt, v in _fields(lst):
                        if vnum == 1:
                            vals.append(np.frombuffer(v, dtype="<f4"))
                    out[name] = np.concatenate(vals) if vals else np.zeros((0,), np.float32)
                elif kind == 3:
                    ints: List[int] = []
                    for vnum, wt, v in _fields(lst):
                        if vnum != 1:
                            continue
                        if wt == 0:
                            ints.append(v)
                        else:
                            p = 0
                            while p < len(v):
                                x, p = _varint(v, p)
                                ints.append(x)
                    out[name] = np.asarray([x - (1 << 64) if x >= (1 << 63) else x for x in ints], np.int64)
                elif kind == 1:
                    out[name] = [v for vnum, _, v in _fields(lst) if vnum == 1]
    return out


def _enc_varint(x: int) -> bytes:
    x &= (1 << 64) - 1
    out = bytearray()
    while True:
        b = x & 0x7F
        x >>= 7
        if x:
            out.append(b | 0x80)
        else:
            out.append(b)
            return bytes(out)


def _ld(num: int, payload: bytes) -> bytes:
    return _enc_varint((num << 3) | 2) + _enc_varint(len(payload)) + payload


def serialize_example(inputs: np.ndarray) -> bytes:
    """tf.train.Example{inputs: FloatList(flattened), input_shape: Int64List} as transform_encoded_data.py writes."""
    flat = np.ascontiguousarray(inputs, dtype="<f4").reshape(-1)
    f_inputs = _ld(2, _ld(1, flat.tobytes()))                                        # Feature.float_list (packed)
    f_shape = _ld(3, _ld(1, b"".join(_enc_varint(int(s)) for s in inputs.shape)))    # Feature.int64_list (packed)
    entries = b"".join(_ld(1, _ld(1, k.encode()) + _ld(2, v)) for k, v in (("inputs", f_inputs), ("input_shape", f_shape)))
    return _ld(1, entries)


# ------------------------------------------------------------------------------------------------ transforms
def load(path: str):
    with open(path, "rb") as f:
        return pickle.load(f)


def save(obj, path: str) -> None:
    os.makedirs(os.path.dirname(path), exist_ok=True)
    with open(path, "wb") as f:
        pickle.dump(obj, f, protocol=4)


def normalize_dataset(batch, data_min, data_max):
    """input_pipeline.py:36-40."""
    batch = (batch - data_min) / (data_max - data_min)
    return 2.0 * batch - 1.0


def slice_transform(batch, problem="vae", slice_idx=None, dim_weights=None):
    """input_pipeline.py:43-48."""
    if dim_weights is not None:
        batch = batch * dim_weights
    if slice_idx is not None:
        batch = np.take(batch, slice_idx, axis=-1)
    return batch


def data_transform(batch, problem="vae", pca=None):
    """input_pipeline.py:51-75 (vae / toy branch)."""
    if pca is not None:
        if batch.ndim > 2:
            shape = batch.shape
            batch = pca.transform(batch.reshape(shape[0], -1)).reshape(*shape)
        else:
            batch = pca.transform(batch)
    return batch


def inverse_data_transform(batch, normalize=True, pca=None, data_min=0.0, data_max=1.0, slice_idx=None,
                           dim_weights=None, out_channels=512):
    """input_pipeline.py:78-110 (un-sliced dimensions are filled with N(0,1) draws, as upstream)."""
    batch = np.asarray(batch)
    if normalize:
        batch = (batch + 1.0) / 2.0
        batch = (data_max - data_min) * batch + data_min
    if pca is not None:
        batch = pca.inverse_transform(batch)
    if slice_idx is not None:
        transformed = np.random.randn(*batch.shape[:-1], out_channels)
        transformed[..., slice_idx] = batch
        batch = transformed
    if dim_weights is not None:
        batch = batch / dim_weights
    return batch


# ------------------------------------------------------------------------------------------------ dataset
class Dataset:
    """Re-iterable stream of float32 batches (B, *shape); attributes min / max / examples like the reference's."""

    def __init__(self, examples_fn, batch_size: int, shuffle: bool, seed: int, transform):
        self._examples_fn = examples_fn
        self.batch_size = batch_size
        self.shuffle = shuffle
        self._seed = seed
        self._epoch = 0
        self._transform = transform
        self.min, self.max = 0.0, 1.0
        self._norm = False

    def _raw_batches(self) -> Iterator[np.ndarray]:
        rng = np.random.default_rng(self._seed + self._epoch)
        self._epoch += 1
        buf: List[np.ndarray] = []
        cap = 8 * self.batch_size if self.shuffle else 1
        pending: List[np.ndarray] = []

        def emit(x):
            pending.append(x)
            if len(pending) == self.batch_size:
                out = np.stack(pending).astype(np.float32)
                pending.clear()
                return out
            return None

        for ex in self._examples_fn(rng if self.shuffle else None):
            if len(buf) < cap:
                buf.append(ex)
                if len(buf) < cap:
                    continue
            j = int(rng.integers(len(buf))) if self.shuffle else 0
            out = emit(buf[j])
            buf[j] = buf[-1]
            buf.pop()
            if out is not None:
                yield out
        while buf:
            j = int(rng.integers(len(buf))) if self.shuffle else 0
            out = emit(buf[j])
            buf[j] = buf[-1]
            buf.pop()
            if out is not None:
                yield out
        # drop_remainder=True: an incomplete final batch is discarded

    def batches_untransformed_norm(self) -> Iterator[np.ndarray]:
        for b in self._raw_batches():
            yield self._transform(b)

    def __iter__(self) -> Iterator[np.ndarray]:
        for b in self.batches_untransformed_norm():
            yield normalize_dataset(b, self.min, self.max).astype(np.float32) if self._norm else b.astype(np.float32)

    def take(self, n: int) -> np.ndarray:
        """The first n examples (fewer if the split is smaller) of the next pass, as iteration yields them.  The pass
        is not used up: the next iteration sees the same order, so reading examples does not change what a later
        evaluation reads."""
        epoch, rows, count = self._epoch, [], 0
        try:
            for b in self:
                rows.append(b)
                count += len(b)
                if count >= n:
                    break
        finally:
            self._epoch = epoch
        return np.concatenate(rows)[:n] if rows else np.zeros((0,), np.float32)


def _tfrecord_examples(pattern: str, shape):
    files = sorted(glob.glob(os.path.expanduser(pattern)))
    if not files:
        raise FileNotFoundError(f"no TFRecord shards match {pattern}")
    n = int(np.prod(shape))

    def gen(rng):
        order = list(files)
        if rng is not None:
            rng.shuffle(order)
        for path in order:
            for payload in read_tfrecord(path):
                ex = parse_example(payload)
                arr = ex["inputs"]
                shp = tuple(int(s) for s in ex.get("input_shape", shape))
                if arr.size != n:
                    raise ValueError(f"{path}: example has {arr.size} values, expected {n} for shape {shape}")
                yield arr.reshape(shp)
    return gen


def _synthetic_examples(shape, count: int, seed: int):
    def gen(rng):
        r = np.random.default_rng(seed)
        for _ in range(count):
            yield r.standard_normal(shape).astype(np.float32)
    return gen


def _save_atomic(obj, path: str) -> None:
    """Write-then-rename: a concurrent reader (another rank under torchrun) never sees a half-written pickle."""
    os.makedirs(os.path.dirname(path), exist_ok=True)
    tmp = f"{path}.tmp.{os.getpid()}"
    save(obj, tmp)
    os.replace(tmp, path)


def _cached_many(paths, compute):
    """Values cached one per pickle in `paths` (utils/data_utils.py:63-156 keeps min / max / cardinality that way).
    `compute()` returns all of them from ONE pass over the data.  Under torch.distributed only rank 0 computes and
    writes; the other ranks wait at a barrier and read what rank 0 wrote, so every rank normalises identically."""
    import torch.distributed as dist
    multi = dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1
    if all(os.path.exists(q) for q in paths):
        return tuple(load(q) for q in paths)
    vals = None
    if not multi or dist.get_rank() == 0:
        vals = tuple(compute())
        try:
            for q, v in zip(paths, vals):
                _save_atomic(v, q)
        except OSError:
            if multi:
                raise
    if multi:
        dist.barrier()
        if vals is None:
            vals = tuple(load(q) for q in paths)
    return vals


class DevicePrefetcher:
    """input_pipeline.py:209-210 (`dataset.prefetch(AUTOTUNE)`) for the GPU path: a background thread pulls host
    batches, stages them in pinned memory and issues the host->device copy on its own CUDA stream, `depth` batches
    ahead of the training step; iteration yields device tensors whose copy the consumer stream has been made to wait
    for.  Without a CUDA device the batches are yielded as they are (host arrays) -- there is nothing to overlap."""

    def __init__(self, dataset, depth: int = 2, device=None):
        self.dataset = dataset
        self.depth = max(1, int(depth))
        self.device = device
        for attr in ("examples", "min", "max", "batch_size"):
            if hasattr(dataset, attr):
                setattr(self, attr, getattr(dataset, attr))

    def __iter__(self):
        import queue
        import threading
        import torch
        if not torch.cuda.is_available():
            yield from self.dataset
            return
        dev = torch.device(self.device or f"cuda:{torch.cuda.current_device()}")
        copy_stream = torch.cuda.Stream(device=dev)
        q: "queue.Queue" = queue.Queue(maxsize=self.depth)
        stop = threading.Event()
        END = object()

        def worker():
            try:
                torch.cuda.set_device(dev)
                for b in self.dataset:
                    if stop.is_set():
                        return
                    host = torch.from_numpy(np.ascontiguousarray(b, np.float32)).pin_memory()
                    with torch.cuda.stream(copy_stream):
                        d = host.to(dev, non_blocking=True)
                        ev = torch.cuda.Event()
                        ev.record(copy_stream)
                    q.put((d, ev, host))        # `host` stays referenced until the consumer has the batch
                q.put(END)
            except BaseException as e:          # surface loader errors in the training thread
                q.put(e)

        th = threading.Thread(target=worker, daemon=True)
        th.start()
        try:
            while True:
                item = q.get()
                if item is END:
                    return
                if isinstance(item, BaseException):
                    raise item
                d, ev, _host = item
                torch.cuda.current_stream().wait_event(ev)
                d.record_stream(torch.cuda.current_stream())
                yield d
        finally:
            # closing the iterator early (a step limit mid-epoch) must not leave the worker inside a CUDA call when the
            # interpreter exits: unblock it from a full queue and wait for it
            stop.set()
            while th.is_alive():
                try:
                    q.get_nowait()
                except queue.Empty:
                    pass
                th.join(timeout=0.01)


def get_dataset(dataset="", data_shape=(2,), problem="vae", batch_size=128, normalize=True, pca_ckpt="",
                slice_ckpt="", dim_weights_ckpt="", include_cardinality=True, synthetic=False,
                synthetic_examples=4096, seed=0):
    """input_pipeline.py:113-235 without TensorFlow.  Returns (train_ds, eval_ds)."""
    if problem == "mnist":
        raise ValueError("problem=mnist is outside the DDPM latent hot path")
    if problem not in ("vae", "toy"):
        raise ValueError(f"Unknown problem type: {problem}")
    shape = tuple(map(int, data_shape))
    pca = load(os.path.expanduser(pca_ckpt)) if pca_ckpt else None
    slice_idx = load(os.path.expanduser(slice_ckpt)) if slice_ckpt else None
    dim_weights = load(os.path.expanduser(dim_weights_ckpt)) if dim_weights_ckpt else None
    if slice_idx is not None:
        slice_idx = np.asarray(slice_idx).astype(np.int64)

    def transform(batch):
        batch = data_transform(batch, problem=problem, pca=pca)
        return slice_transform(batch, problem=problem, slice_idx=slice_idx, dim_weights=dim_weights)

    out = []
    for split, sd in (("train", 0), ("eval", 1)):
        if synthetic:
            gen = _synthetic_examples(shape, synthetic_examples if split == "train" else max(batch_size, synthetic_examples // 8),
                                      seed * 2 + sd)
        else:
            gen = _tfrecord_examples(f"{dataset}/{split}-*.tfrecord", shape)
        ds = Dataset(gen, batch_size, shuffle=True, seed=seed * 2 + sd, transform=transform)
        cache_dir = os.path.join(os.path.expanduser(dataset), "cache") if (dataset and not synthetic) else None
        if normalize:
            config = "".join(p.split("/")[-1].split(".")[0] for p in (pca_ckpt, slice_ckpt, dim_weights_ckpt))

            def minmax(ds=ds):
                lo, hi = np.float32(np.finfo(np.float32).max), np.float32(np.finfo(np.float32).min)
                for b in ds.batches_untransformed_norm():
                    lo, hi = min(lo, np.float32(b.min())), max(hi, np.float32(b.max()))
                return lo, hi
            if cache_dir:
                lo, hi = _cached_many([os.path.join(cache_dir, f"{split}_{config}_min.pkl"),
                                       os.path.join(cache_dir, f"{split}_{config}_max.pkl")], minmax)   # one pass
            else:
                lo, hi = minmax()
            ds.min, ds.max, ds._norm = lo, hi, True
        if include_cardinality:
            def count(ds=ds):
                return sum(1 for _ in ds._raw_batches())
            ds.examples = (_cached_many([os.path.join(cache_dir, f"{split}_{batch_size}_cardinality.pkl")],
                                        lambda: (count(),))[0] if cache_dir else count())
        out.append(ds)
    return out[0], out[1]
