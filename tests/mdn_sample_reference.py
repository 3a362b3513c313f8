"""CPU restatement of the reference's autoregressive sampler (sample_mdn.py:54-119), next to tests/mdn_reference.py.

The random-number recipe is an ASSUMPTION about tfp-nightly 0.12.0.dev20201127 on jax 0.2.8 (the reference's pins),
which cannot run here to confirm it:
  MixtureSameFamily._sample_n: components_seed, mix_seed = split_seed(seed, salt='MixtureSameFamily')
                                                        = split(fold_in(seed, MIXTURE_SALT))
  Categorical(logits=pi).sample: jax.random.categorical = argmax(pi + gumbel(mix_key, (R, Kc)))  (first index on ties)
  MultivariateNormalDiag(mu, sigma).sample: mu + sigma * normal(comp_key, (R, Kc, C)), read at the chosen component
The C++ host function mdn_mixture_keys (csrc/mdn.cu) states the same key derivation, so a correction touches those two
places and no kernel.
"""
from __future__ import annotations

import numpy as np

from oracle import threefry as TF

MIXTURE_SALT = 0x916F26AB   # int(hashlib.sha512(b"MixtureSameFamily").hexdigest(), 16) & 0xFFFFFFFF
_F32_TINY = np.finfo(np.float32).tiny


def fold_in(key, data: int) -> np.ndarray:
    """jax 0.2.8 random.fold_in: threefry_2x32(key, threefry_seed(data)) = the threefry block of key on (0, data)."""
    x0, x1 = TF.threefry2x32_block(key[0], key[1], np.uint32(0), np.uint32(data & 0xFFFFFFFF))
    return np.array([x0, x1], dtype=np.uint32)


def mixture_sample_keys(key):
    """(components key, mixture key) of MixtureSameFamily(...).sample(seed=key)."""
    comp, mix = TF.split(fold_in(key, MIXTURE_SALT), 2)
    return comp, mix


def random_bits_at(key, idx: np.ndarray, n: int) -> np.ndarray:
    """Elements idx of jax.random._random_bits(key, 32, (n,)) without generating the other n - len(idx)."""
    idx = np.asarray(idx, np.int64)
    half = (n + 1) // 2
    lo = idx < half
    x0 = np.where(lo, idx, idx - half)
    x1 = np.where(lo, idx + half, idx)
    x1 = np.where(x1 >= n, 0, x1)          # odd n: the pad counter is 0
    o0, o1 = TF.threefry2x32_block(key[0], key[1], x0.astype(np.uint32), x1.astype(np.uint32))
    return np.where(lo, o0, o1).astype(np.uint32)


def _u01(bits):
    return (((bits >> np.uint32(9)) | np.uint32(0x3F800000)).view(np.float32) - np.float32(1.0)).astype(np.float32)


def mixture_sample(pi, mu, log_sigma, key, first_row: int = 0, total_rows: int = 0, row_index=None):
    """Rows of MixtureSameFamily(Categorical(logits=pi), MultivariateNormalDiag(mu, exp(log_sigma))).sample(seed=key),
    float32: pi (rows, Kc), mu / log_sigma (rows, Kc*C) -> (x (rows, C), k* (rows,)).  Local row j is row
    first_row + j of a draw over total_rows rows (0: rows), or row row_index[j] when given."""
    pi = np.asarray(pi, np.float32)
    rows, kc = pi.shape
    mu = np.asarray(mu, np.float32).reshape(rows, kc, -1)
    ls = np.asarray(log_sigma, np.float32).reshape(rows, kc, -1)
    C = mu.shape[-1]
    total = total_rows or rows
    r = np.arange(rows, dtype=np.int64) + first_row if row_index is None else np.asarray(row_index, np.int64)
    comp_key, mix_key = mixture_sample_keys(key)
    u01 = _u01(random_bits_at(mix_key, r[:, None] * kc + np.arange(kc), total * kc))
    tiny = np.float32(_F32_TINY)
    u = np.maximum(tiny, (u01 * (np.float32(1.0) - tiny) + tiny).astype(np.float32))
    with np.errstate(divide="ignore"):
        g = (-np.log(-np.log(u))).astype(np.float32)
    k = np.argmax((pi + g).astype(np.float32), axis=-1)
    bits = random_bits_at(comp_key, ((r * kc + k) * C)[:, None] + np.arange(C), total * kc * C)
    lo = np.nextafter(np.float32(-1.0), np.float32(0.0))
    uz = np.maximum(lo, (_u01(bits) * (np.float32(1.0) - lo) + lo).astype(np.float32))
    z = (np.float32(np.sqrt(2)) * TF.erfinv_f32(uz)).astype(np.float32)
    sel = np.arange(rows)
    x = (mu[sel, k] + (np.exp(ls[sel, k]).astype(np.float32) * z).astype(np.float32)).astype(np.float32)
    return x, k


def step_keys(key, steps: int):
    """embed_rng of each decoding step: rng, embed_rng = split(rng) (sample_mdn.py:109), from the rng left after the
    model_rng split."""
    rng, out = np.asarray(key, np.uint32), []
    for _ in range(steps):
        rng, embed = TF.split(rng, 2)
        out.append(embed)
    return out


def sample_mdn(model, key, n: int, S: int, C: int, first_row: int = 0, total_rows: int = 0):
    """sample_mdn.py:89-117 with model(tokens) -> (pi, mu, log_sigma) as float32 arrays (the shift=False forward).
    Returns (tokens, chain): the reference's result and the tokens before the last step."""
    tokens = np.zeros((n, S, C), np.float32)
    total = (total_rows or n) * S
    rows = (first_row * S + np.arange(n * S)).astype(np.int64)
    chain = None
    for i, ek in enumerate(step_keys(key, S)):
        pi, mu, ls = (np.asarray(a, np.float32).reshape(n * S, -1) for a in model(tokens))
        nxt, _ = mixture_sample(pi, mu, ls, ek, total_rows=total, row_index=rows)
        nxt = nxt.reshape(n, S, C)
        if i < S - 1:
            tokens[:, i + 1] = nxt[:, i]
        else:
            chain = tokens.copy()
            tokens = nxt
    return tokens, chain
