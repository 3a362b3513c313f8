"""Float64 restatements of the single steps of the hand-written backward pass.

Each function is the adjoint of ONE forward operation of oracle/ddpm_oracle.py (SURVEY Appendix E), written from the
math, taking that operation's saved inputs and the adjoint of its output and returning the adjoints of its inputs and
parameters.  tests/test_gpu_backward_stages.py feeds them with the operands one kernel launch read from device memory
and compares with what that launch wrote; tests/test_backward_reference.py checks every function against
torch.autograd through the oracle's forward functions, so a wrong restatement cannot hide behind a matching wrong
kernel.  Everything is plain torch; callers pass float64 tensors (on any device).
"""
from __future__ import annotations

import math

import torch

Tensor = torch.Tensor

LN_EPS = 1e-6


# ----------------------------------------------------------------------------------------------------------------
# bfloat16 storage
# ----------------------------------------------------------------------------------------------------------------
def bf16_round(x: Tensor) -> Tensor:
    """x rounded to the nearest bfloat16 (ties to even), returned in x's dtype."""
    return x.to(torch.float32).to(torch.bfloat16).to(x.dtype)


def bf16_ulp(x: Tensor) -> Tensor:
    """Spacing of the bfloat16 numbers around x (8 significant bits); the smallest normal spacing near zero."""
    _, e = torch.frexp(x.abs().clamp_min(2.0 ** -126))   # |x| = m 2^e with m in [0.5, 1)
    return torch.ldexp(torch.ones_like(x), e - 8)


# ----------------------------------------------------------------------------------------------------------------
# dense layers: y = x @ W + b with W stored (in, out)
# ----------------------------------------------------------------------------------------------------------------
def dense_bwd_w(x: Tensor, g: Tensor) -> Tensor:
    """dL/dW = x^T g over all rows."""
    return x.reshape(-1, x.shape[-1]).T @ g.reshape(-1, g.shape[-1])


def dense_bwd_x(g: Tensor, w: Tensor) -> Tensor:
    """dL/dx = g W^T."""
    return g @ w.T


def dense_bwd_b(g: Tensor) -> Tensor:
    """dL/db = column sums of g."""
    return g.reshape(-1, g.shape[-1]).sum(dim=0)


# ----------------------------------------------------------------------------------------------------------------
# activations
# ----------------------------------------------------------------------------------------------------------------
def gelu_tanh_grad(x: Tensor) -> Tensor:
    """d/dx of 0.5 x (1 + tanh(c (x + 0.044715 x^3))), c = sqrt(2 / pi)."""
    c = math.sqrt(2.0 / math.pi)
    t = torch.tanh(c * (x + 0.044715 * x ** 3))
    return 0.5 * (1.0 + t) + 0.5 * x * (1.0 - t * t) * c * (1.0 + 3.0 * 0.044715 * x * x)


def swish_grad(x: Tensor) -> Tensor:
    """d/dx of x sigmoid(x)."""
    s = torch.sigmoid(x)
    return s * (1.0 + x * (1.0 - s))


# ----------------------------------------------------------------------------------------------------------------
# LayerNorm (flax 0.3.0: var = E[x^2] - E[x]^2, eps 1e-6), optionally followed by FiLM and swish
# ----------------------------------------------------------------------------------------------------------------
def row_stats(x: Tensor) -> Tensor:
    """(sum, sum of squares) of every row: the form in which the wide LayerNorms keep their statistics."""
    return torch.stack([x.sum(dim=-1), (x * x).sum(dim=-1)], dim=-1)


def layer_norm_bwd(g: Tensor, x: Tensor, gamma: Tensor, stats: Tensor | None = None):
    """Adjoint of y = (x - mean) rsqrt(var + eps) gamma + beta.  stats: per-row (sum, sumsq) to take mean and variance
    from, else they are computed from x.  Returns dx, dgamma, dbeta."""
    n = x.shape[-1]
    st = row_stats(x) if stats is None else stats
    mean = (st[..., 0] / n).unsqueeze(-1)
    rstd = torch.rsqrt(st[..., 1].unsqueeze(-1) / n - mean * mean + LN_EPS)
    xh = (x - mean) * rstd
    dxh = g * gamma
    dx = rstd * (dxh - dxh.mean(dim=-1, keepdim=True) - xh * (dxh * xh).mean(dim=-1, keepdim=True))
    flat = lambda t: t.reshape(-1, n)
    return dx, flat(g * xh).sum(dim=0), flat(g).sum(dim=0)


def ln_film_swish_bwd(g: Tensor, x: Tensor, gamma: Tensor, beta: Tensor, scale: Tensor, shift: Tensor,
                      stats: Tensor | None = None):
    """Adjoint of out = swish(scale * LayerNorm(x) + shift) (models/shared.py:62-64): x, g are (B, S, N); scale, shift
    (B, N), one pair per example.  Returns dx, dgamma, dbeta, dscale, dshift (the last two (B, N))."""
    n = x.shape[-1]
    st = row_stats(x) if stats is None else stats
    mean = (st[..., 0] / n).unsqueeze(-1)
    rstd = torch.rsqrt(st[..., 1].unsqueeze(-1) / n - mean * mean + LN_EPS)
    y = (x - mean) * rstd * gamma + beta
    sc, sh = scale[:, None, :], shift[:, None, :]
    dz = g * swish_grad(sc * y + sh)
    dx, dgamma, dbeta = layer_norm_bwd(dz * sc, x, gamma, st)
    return dx, dgamma, dbeta, (dz * y).sum(dim=1), dz.sum(dim=1)


def ssm_ln_film_swish_bwd(g: Tensor, gt: Tensor, x: Tensor, xt: Tensor, gamma: Tensor, beta: Tensor,
                          scale: Tensor | None = None, shift: Tensor | None = None, stats: Tensor | None = None,
                          act: str | None = "swish"):
    """Sliced score matching's reverse pass through out = act(scale * LayerNorm(x) + shift) AND its tangent
    out' = J_out(x) x': the gradient of <g, out> + <g', out'> with respect to x, x', gamma, beta, scale and shift.

    Conventions as ln_film_swish_bwd: x, xt, g, gt are (B, S, N) with one FiLM pair (B, N) per example; scale=None is a
    plain LayerNorm; act is "swish" or None; mean and variance take the values of the (sum, sumsq) stats.  Derived by
    float64 autograd, not from the kernel's closed form: out' is the JVP of out (double-vjp), and the statistics carry
    the stats' values while differentiating as functions of x.  Returns dx, dxt, dgamma, dbeta, dscale, dshift (the
    last two (B, N), or None without FiLM)."""
    n = x.shape[-1]
    st = row_stats(x) if stats is None else stats
    m_dev = (st[..., 0] / n).unsqueeze(-1)
    v_dev = st[..., 1].unsqueeze(-1) / n - m_dev * m_dev
    film = scale is not None
    with torch.enable_grad():
        leaves = [t.detach().clone().requires_grad_(True) for t in (x, xt, gamma, beta)]
        if film:
            leaves += [t.detach().clone().requires_grad_(True) for t in (scale, shift)]
        xl, xtl, gl, bl = leaves[:4]
        m_live = xl.mean(dim=-1, keepdim=True)
        v_live = (xl * xl).mean(dim=-1, keepdim=True) - m_live * m_live
        mean = m_live + (m_dev - m_live).detach()
        var = v_live + (v_dev - v_live).detach()
        z = (xl - mean) * torch.rsqrt(var + LN_EPS) * gl + bl
        if film:
            z = leaves[4][:, None, :] * z + leaves[5][:, None, :]
        out = z * torch.sigmoid(z) if act == "swish" else z
        w = torch.zeros_like(out, requires_grad=True)
        vjp, = torch.autograd.grad(out, xl, w, create_graph=True)
        out_t, = torch.autograd.grad(vjp, w, xtl, create_graph=True)
        obj = (g * out).sum() + (gt * out_t).sum()
        grads = torch.autograd.grad(obj, leaves, allow_unused=True)
    grads = [torch.zeros_like(leaf) if d is None else d.detach() for d, leaf in zip(grads, leaves)]
    dx, dxt, dgamma, dbeta = grads[:4]
    dgamma, dbeta = dgamma.reshape(n), dbeta.reshape(n)
    return (dx, dxt, dgamma, dbeta) + (tuple(grads[4:]) if film else (None, None))


# ----------------------------------------------------------------------------------------------------------------
# multi-head attention core (q scaled by 1 / sqrt(depth) before the dot product)
# ----------------------------------------------------------------------------------------------------------------
def attention_bwd(qkv: Tensor, probs: Tensor, d_out: Tensor, num_heads: int) -> Tensor:
    """qkv (B, S, 3E) = [q | k | v], head-major inside each E block; probs (B, H, S, S) the softmax weights of the
    forward pass; d_out (B, S, E) the adjoint of the concatenated head outputs.  Returns d qkv (B, S, 3E)."""
    B, S, E3 = qkv.shape
    E = E3 // 3
    dh = E // num_heads
    q, k, v = (t.reshape(B, S, num_heads, dh) for t in qkv.split(E, dim=-1))
    do = d_out.reshape(B, S, num_heads, dh)
    qs = 1.0 / math.sqrt(dh)
    dp = torch.einsum("bqhd,bkhd->bhqk", do, v)
    ds = probs * (dp - (dp * probs).sum(dim=-1, keepdim=True))
    dv = torch.einsum("bhqk,bqhd->bkhd", probs, do)
    dq = torch.einsum("bhqk,bkhd->bqhd", ds, k) * qs
    dk = torch.einsum("bhqk,bqhd->bkhd", ds, q) * qs
    return torch.cat([dq.reshape(B, S, E), dk.reshape(B, S, E), dv.reshape(B, S, E)], dim=-1)


# ----------------------------------------------------------------------------------------------------------------
# FiLM generator (models/ncsn.py:47-61): enc -> d1 -> swish -> d2 -> ss = [scale | shift]
# ----------------------------------------------------------------------------------------------------------------
def film_generator_bwd(dss: Tensor, enc: Tensor, e1pre: Tensor, e1: Tensor, e2: Tensor, w_ss: Tensor, w_d2: Tensor):
    """dss (B, 2N): adjoint of [scale | shift]; enc (B, 128) the noise encoding (no gradient flows into it);
    e1pre = enc W1 + b1, e1 = swish(e1pre), e2 = e1 W2 + b2 the saved activations.  Returns a dict with the six parameter
    gradients and the two intermediate adjoints de2, de1."""
    de2 = dense_bwd_x(dss, w_ss)
    de1 = dense_bwd_x(de2, w_d2) * swish_grad(e1pre)
    return {"ss.kernel": dense_bwd_w(e2, dss), "ss.bias": dense_bwd_b(dss),
            "d2.kernel": dense_bwd_w(e1, de2), "d2.bias": dense_bwd_b(de2),
            "d1.kernel": dense_bwd_w(enc, de1), "d1.bias": dense_bwd_b(de1),
            "de2": de2, "de1": de1}


# ----------------------------------------------------------------------------------------------------------------
# objectives: per-example loss and d(mean over the global batch of the loss) / d(network output)
# ----------------------------------------------------------------------------------------------------------------
def ddpm_loss_seed(eps: Tensor, pred: Tensor, global_batch: int):
    """utils/losses.py:304-308: loss_b = mean over the example of (eps - pred)^2.  Returns (loss (B,), dpred)."""
    B = eps.shape[0]
    per = eps[0].numel()
    d = eps - pred
    return (d * d).reshape(B, -1).mean(dim=1), -2.0 * d / (global_batch * per)


def dsm_loss_seed(eps: Tensor, raw: Tensor, global_batch: int):
    """utils/losses.py:161-179 for a network whose score is raw / sigma: the target is -eps / sigma, so
    loss_b = 0.5 sigma^2 sum((raw + eps)^2 / sigma^2) = 0.5 sum((raw + eps)^2).  Returns (loss (B,), draw)."""
    B = eps.shape[0]
    d = raw + eps
    return 0.5 * (d * d).reshape(B, -1).sum(dim=1), d / global_batch
