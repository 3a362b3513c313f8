"""Float64 restatements of the single launches of the hand-written forward pass.

Each function takes the operands ONE kernel launch reads and returns what that launch should have written, written
from the math of oracle/ddpm_oracle.py.  tests/test_gpu_forward_stages.py feeds them with the operands a launch read
from device memory and compares with what it wrote; tests/test_forward_reference.py composes them back into the
oracle's networks, so a wrong restatement cannot agree with a wrong kernel unnoticed.  Everything is plain torch;
callers pass float64 tensors (on any device).  The bfloat16 helpers and the row statistics are those of the backward
restatements.
"""
from __future__ import annotations

import math

import torch

from tests.backward_reference import LN_EPS, bf16_round, bf16_ulp, row_stats  # noqa: F401  (re-exported)

Tensor = torch.Tensor


# ----------------------------------------------------------------------------------------------------------------
# activations and LayerNorm (flax 0.3.0: var = E[x^2] - E[x]^2, eps 1e-6)
# ----------------------------------------------------------------------------------------------------------------
def gelu_tanh(x: Tensor) -> Tensor:
    """0.5 x (1 + tanh(c (x + 0.044715 x^3))), c = sqrt(2 / pi)."""
    return 0.5 * x * (1.0 + torch.tanh(math.sqrt(2.0 / math.pi) * (x + 0.044715 * x ** 3)))


def swish(x: Tensor) -> Tensor:
    return x * torch.sigmoid(x)


def layer_norm(x: Tensor, gamma: Tensor, beta: Tensor, stats: Tensor | None = None) -> Tensor:
    """(x - mean) rsqrt(var + eps) gamma + beta over the last axis; stats: per-row (sum, sumsq) to take mean and
    variance from (the form the wide LayerNorms receive them in), else computed from x."""
    n = x.shape[-1]
    st = row_stats(x) if stats is None else stats
    mean = (st[..., 0] / n).unsqueeze(-1)
    rstd = torch.rsqrt(st[..., 1].unsqueeze(-1) / n - mean * mean + LN_EPS)
    return (x - mean) * rstd * gamma + beta


# ----------------------------------------------------------------------------------------------------------------
# trunk launches
# ----------------------------------------------------------------------------------------------------------------
def embed(x: Tensor, w_in: Tensor, b_in: Tensor, posenc: Tensor, gamma: Tensor, beta: Tensor):
    """x (B, S, C) -> h = x W_in + b_in + posenc[s] (B, S, 128) and a = LayerNorm(h)."""
    h = x @ w_in + b_in + posenc[: x.shape[-2]]
    return h, layer_norm(h, gamma, beta)


def gemm(a: Tensor, w: Tensor, bias: Tensor | None = None, residual: Tensor | None = None, act: str | None = None,
         ln: tuple | None = None):
    """One forward GEMM with its epilogue: v = a w (+ bias) (+ residual).  Returns a dict with "v" (the fp32 output /
    the pre-activation), "act" (gelu_tanh(v) when act == "gelu"), "ln" (LayerNorm(v; *ln) when ln = (gamma, beta))
    and "stats" (the row (sum, sumsq) of v)."""
    v = a @ w
    if bias is not None:
        v = v + bias
    if residual is not None:
        v = v + residual
    out = {"v": v, "stats": row_stats(v)}
    if act == "gelu":
        out["act"] = gelu_tanh(v)
    elif act is not None:
        raise ValueError(act)
    if ln is not None:
        out["ln"] = layer_norm(v, *ln)
    return out


def attention(qkv: Tensor, num_heads: int, causal: bool = False):
    """qkv (B, S, 3E) = [q | k | v], head-major inside each E block; q scaled by 1 / sqrt(dh) before the dot product.
    Returns (probs (B, H, S, S), o (B, S, E)); causal: probabilities above the diagonal are exactly zero."""
    B, S, E3 = qkv.shape
    E = E3 // 3
    dh = E // num_heads
    q, k, v = (t.reshape(B, S, num_heads, dh) for t in qkv.split(E, dim=-1))
    logits = torch.einsum("bqhd,bkhd->bhqk", q / math.sqrt(dh), k)
    if causal:
        mask = torch.ones(S, S, dtype=torch.bool, device=qkv.device).triu(1)
        logits = logits.masked_fill(mask, -math.inf)
    probs = torch.softmax(logits, dim=-1)
    o = torch.einsum("bhqk,bkhd->bqhd", probs, v).reshape(B, S, E)
    return probs, o


def attn_block(a: Tensor, h_in: Tensor, w_qkv: Tensor, b_qkv: Tensor, w_o: Tensor, b_o: Tensor, gamma: Tensor,
               beta: Tensor, num_heads: int, round_o: bool = True):
    """The fused attention block: h_mid = attention(a W_qkv + b_qkv) W_o + b_o + h_in, a2 = LayerNorm(h_mid).  a, h_in
    (B, S, 128).  The attention output o exists only on chip, as the bf16 operand of the out-projection: round_o
    rounds the restatement's own o to bf16 as the kernel does.  Returns (h_mid, a2)."""
    _, o = attention(a @ w_qkv + b_qkv, num_heads)
    if round_o:
        o = bf16_round(o)
    h_mid = o @ w_o + b_o + h_in
    return h_mid, layer_norm(h_mid, gamma, beta)


def ffn_fused(a2: Tensor, h_mid: Tensor, w1: Tensor, b1: Tensor, w2: Tensor, b2: Tensor, gamma: Tensor, beta: Tensor,
              round_hidden: bool = True):
    """The fused FFN: h_out = gelu(a2 W1 + b1) W2 + b2 + h_mid, a_next = LayerNorm(h_out).  The hidden activation
    exists only on chip, as a bf16 operand: round_hidden rounds the restatement's own to bf16.  Returns
    (h_out, a_next)."""
    hid = gelu_tanh(a2 @ w1 + b1)
    if round_hidden:
        hid = bf16_round(hid)
    h_out = hid @ w2 + b2 + h_mid
    return h_out, layer_norm(h_out, gamma, beta)


# ----------------------------------------------------------------------------------------------------------------
# FiLM'd residual tail
# ----------------------------------------------------------------------------------------------------------------
def film_rows(ss: Tensor, M: int, S: int, broadcast: bool = False, row: int | None = None) -> Tensor:
    """The (M, 2N) FiLM row of every LayerNorm row: row m of a per-example table ss (B, 2N) is m // S; broadcast: row 0
    for all; row: that explicit row of the table (the sampler's FiLM table)."""
    if row is not None:
        return ss[row].expand(M, -1)
    if broadcast:
        return ss[0].expand(M, -1)
    return ss.repeat_interleave(S, dim=0)[:M]


def ln_film_act(u: Tensor, stats: Tensor | None, gamma: Tensor, beta: Tensor, rows: Tensor | None, act: bool):
    """One ln_film_act launch: out = swish(scale * LayerNorm(u; stats) + shift) (act) or LayerNorm(u; stats).  u (M, N);
    rows (M, 2N) = [scale | shift] per row (see film_rows), or None (no FiLM).  Returns (out, z) with z the
    pre-activation."""
    n = u.shape[-1]
    z = layer_norm(u, gamma, beta, stats)
    if rows is not None:
        z = rows[:, :n] * z + rows[:, n:]
    return (swish(z) if act else z), z


def noise_encoding(t: Tensor, freqs: Tensor) -> Tensor:
    """enc[r] = [sin(arg) | cos(arg)], arg = (5000 t_r) f_j.  The caller decides in which precision arg is formed: the
    device forms it in float32 (pass arg32=True to film_generator)."""
    arg = (5000.0 * t)[:, None] * freqs[None, :]
    return torch.cat([torch.sin(arg), torch.cos(arg)], dim=1)


def noise_arg_f32(t: Tensor, freqs: Tensor) -> Tensor:
    """(5000 t) f in float32, product by product in that order (as jnp and the kernel round it), back in t's dtype."""
    t32, f32 = t.to(torch.float32), freqs.to(torch.float32)
    return ((5000.0 * t32)[:, None] * f32[None, :]).to(t.dtype)


def film_generator(t: Tensor, freqs: Tensor, p: dict, arg32: bool = True):
    """DenseFiLM: enc = noise_encoding(t); e1pre = enc W1 + b1; e1 = swish(e1pre); e2 = e1 W2 + b2; ss = e2 Wss + bss.
    p holds d1.kernel / d1.bias / d2.kernel / d2.bias / ss.kernel / ss.bias.  Returns a dict of the five tensors."""
    if arg32:
        arg = noise_arg_f32(t, freqs)
        enc = torch.cat([torch.sin(arg), torch.cos(arg)], dim=1)
    else:
        enc = noise_encoding(t, freqs)
    e1pre = enc @ p["d1.kernel"] + p["d1.bias"]
    e1 = swish(e1pre)
    e2 = e1 @ p["d2.kernel"] + p["d2.bias"]
    return {"enc": enc, "e1pre": e1pre, "e1": e1, "e2": e2, "ss": e2 @ p["ss.kernel"] + p["ss.bias"]}


def ln_film_tangent(x: Tensor, stats: Tensor, xt: Tensor, gamma: Tensor, beta: Tensor, rows: Tensor | None,
                    act: bool) -> Tensor:
    """Tangent of out = act(film(LayerNorm(x))) along xt, with mean and rstd from the PRIMAL row statistics (kernels.cuh):
    xh = (x - mean) rstd, xh' = rstd (xt - mean(xt) - xh mean(xh xt)), y' = gamma xh', z' = scale y',
    out' = swish'(z) z' (act) or z'."""
    n = x.shape[-1]
    mean = (stats[..., 0] / n).unsqueeze(-1)
    rstd = torch.rsqrt(stats[..., 1].unsqueeze(-1) / n - mean * mean + LN_EPS)
    xh = (x - mean) * rstd
    xh_t = rstd * (xt - xt.mean(dim=-1, keepdim=True) - xh * (xh * xt).mean(dim=-1, keepdim=True))
    z, zt = gamma * xh + beta, gamma * xh_t
    if rows is not None:
        z, zt = rows[:, :n] * z + rows[:, n:], rows[:, :n] * zt
    if act:
        s = torch.sigmoid(z)
        zt = zt * s * (1.0 + z * (1.0 - s))
    return zt


def scale_rows(y: Tensor, sigma: Tensor) -> Tensor:
    """DenseNCSN's output = y / sigma, one sigma per example (B, ...) ."""
    return y / sigma.reshape((-1,) + (1,) * (y.dim() - 1))


# ----------------------------------------------------------------------------------------------------------------
# per-element bound of a bf16 output computed through tanh.approx.f32
# ----------------------------------------------------------------------------------------------------------------
def activation_excess(got: Tensor, ref: Tensor, pre: Tensor, slack: float = 0.0) -> Tensor:
    """(|got - ref| - ulp_bf16(ref) / 2 - slack) / |pre| per element: the part of the error of an activation stored as
    bf16 that its rounding does not explain, per unit of pre-activation.  slack: an absolute allowance for the fp32
    rounding of the pre-activation itself, which the activation passes on with a slope of about one and which the
    division by a tiny |pre| would otherwise magnify.  swish(v) = h + h tanh(h) with h = v / 2 and
    gelu(v) = h + h tanh(u) with h = v / 2, so an absolute error e of tanh gives |v| e / 2: a tanh good to 2^-11
    keeps this below 2^-12."""
    spacing = bf16_ulp(torch.maximum(ref.abs(), got.abs()))
    return ((got - ref).abs() - 0.5 * spacing - slack).clamp_min(0.0) / pre.abs().clamp_min(1e-30)
