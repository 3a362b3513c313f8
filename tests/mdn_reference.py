"""CPU restatement (torch, fp32 / fp64) of the reference's autoregressive baseline, next to the DDPM oracle whose
primitives it reuses: models/autoregressive.py:25-82 (shift_right, TransformerMDN) and train_mdn.py:100-133 (mdn_loss).

``emulate_bf16=True`` rounds the GEMM operands to bfloat16 where the CUDA path feeds the tensor cores, as in the oracle.
"""
from __future__ import annotations

import math
from typing import Dict

import torch

from oracle import ddpm_oracle as O

Tensor = torch.Tensor


def shift_right(x: Tensor) -> Tensor:
    """models/autoregressive.py:25-33: pad one zero position in front of axis 1, drop the last one."""
    return torch.cat([torch.zeros_like(x[:, :1]), x[:, :-1]], dim=1)


def self_attention(x: Tensor, p: Dict[str, Tensor], prefix: str, num_heads: int, causal: bool = False,
                   emulate_bf16: bool = False) -> Tensor:
    """flax.nn.SelfAttention with ``causal_mask``: the masked logits get a -1e10 bias (flax make_causal_mask +
    attention bias), which the softmax turns into exact zeros."""
    B, S, E = x.shape
    dh = E // num_heads
    qkv = O.dense(x, p[prefix + "qkv.kernel"], p[prefix + "qkv.bias"], emulate_bf16)
    q, k, v = qkv.split(E, dim=-1)
    q = q.reshape(B, S, num_heads, dh) / math.sqrt(dh)
    k = k.reshape(B, S, num_heads, dh)
    v = v.reshape(B, S, num_heads, dh)
    logits = torch.einsum("bqhd,bkhd->bhqk", q, k)
    if causal:
        mask = torch.ones(S, S, dtype=torch.bool).tril()
        logits = logits + torch.where(mask, 0.0, -1e10).to(logits.dtype)
    w = torch.exp(logits - torch.logsumexp(logits, dim=-1, keepdim=True))
    o = torch.einsum("bhqk,bkhd->bqhd", w, v).reshape(B, S, E)
    return O.dense(o, p[prefix + "out.kernel"], p[prefix + "out.bias"], emulate_bf16)


def transformer_mdn(p: Dict[str, Tensor], inputs: Tensor, shift: bool = True, num_layers: int = 6,
                    num_heads: int = 8, num_mlp_layers: int = 2, mlp_dims: int = 2048, mdn_components: int = 100,
                    emulate_bf16: bool = False):
    """models/autoregressive.py:40-82 (TransformerMDN.apply) -> (pi, mu, log_sigma)."""
    B, S, C = inputs.shape
    x = shift_right(inputs) if shift else inputs
    x = O.dense(x, p["in.kernel"], p["in.bias"]) + O.transformer_positional_encoding(S, 128, inputs.dtype)[None]
    for l in range(num_layers):
        pre = f"l{l}."
        a = O.layer_norm(x, p[pre + "ln1.scale"], p[pre + "ln1.bias"])
        x = self_attention(a, p, pre + "attn.", num_heads, True, emulate_bf16) + x
        m = O.layer_norm(x, p[pre + "ln2.scale"], p[pre + "ln2.bias"])
        m = O.gelu_tanh(O.dense(m, p[pre + "ffn1.kernel"], p[pre + "ffn1.bias"], emulate_bf16))
        x = O.dense(m, p[pre + "ffn2.kernel"], p[pre + "ffn2.bias"], emulate_bf16) + x
    x = O.layer_norm(x, p["post_ln.scale"], p["post_ln.bias"])
    x = O.dense(x, p["post.kernel"], p["post.bias"], emulate_bf16)
    for k in range(num_mlp_layers):   # DenseResBlock(x, mlp_dims): scale 1, shift 0
        x = O.dense_res_block(x, 1.0, 0.0, p, f"k{k}.res.", emulate_bf16)
    x = O.layer_norm(x, p["out_ln.scale"], p["out_ln.bias"])
    mu = O.dense(x, p["mdn.mu.kernel"], p["mdn.mu.bias"], emulate_bf16)
    log_sigma = O.dense(x, p["mdn.log_sigma.kernel"], p["mdn.log_sigma.bias"], emulate_bf16)
    pi = O.dense(x, p["mdn.pi.kernel"], p["mdn.pi.bias"], emulate_bf16)
    return pi, mu, log_sigma


def mdn_nll(pi: Tensor, mu: Tensor, log_sigma: Tensor, x: Tensor) -> Tensor:
    """train_mdn.py:100-133 with reduction 'none': -log p(x) under MixtureSameFamily(Categorical(logits=pi),
    MultivariateNormalDiag(mu, exp(log_sigma))); one value per row of x.reshape(-1, C)."""
    C = x.shape[-1]
    kc = pi.shape[-1]
    pi = pi.reshape(-1, kc)
    mu = mu.reshape(-1, kc, C)
    ls = log_sigma.reshape(-1, kc, C)
    x = x.reshape(-1, 1, C)
    z = (x - mu) * torch.exp(-ls)
    comp = (-0.5 * z * z - ls).sum(-1) - 0.5 * C * math.log(2 * math.pi)
    return -torch.logsumexp(torch.log_softmax(pi, dim=-1) + comp, dim=-1)


def mdn_nll_grads(pi: Tensor, mu: Tensor, log_sigma: Tensor, x: Tensor):
    """Closed-form d loss_r / d (pi, mu, log_sigma) per row (what the CUDA kernel writes, unscaled)."""
    C = x.shape[-1]
    kc = pi.shape[-1]
    pi = pi.reshape(-1, kc)
    mu = mu.reshape(-1, kc, C)
    ls = log_sigma.reshape(-1, kc, C)
    inv = torch.exp(-ls)
    z = (x.reshape(-1, 1, C) - mu) * inv
    comp = (-0.5 * z * z - ls).sum(-1) - 0.5 * C * math.log(2 * math.pi)
    lp = torch.log_softmax(pi, dim=-1) + comp
    gam = torch.softmax(lp, dim=-1)
    dmu = -gam[..., None] * z * inv
    dls = gam[..., None] * (1 - z * z)
    dpi = torch.softmax(pi, dim=-1) - gam
    return dpi, dmu.reshape(-1, kc * C), dls.reshape(-1, kc * C)


def param_shapes(C: int, num_layers: int, mlp_dims: int, num_mlp_layers: int, mdn_components: int):
    """Arena tensors of a TransformerMDN plan, in order (name -> shape)."""
    E, Md = 128, mlp_dims
    out = {"in.kernel": (C, E), "in.bias": (E,)}
    for l in range(num_layers):
        pre = f"l{l}."
        out.update({pre + "ln1.scale": (E,), pre + "ln1.bias": (E,), pre + "attn.qkv.kernel": (E, 3 * E),
                    pre + "attn.qkv.bias": (3 * E,), pre + "attn.out.kernel": (E, E), pre + "attn.out.bias": (E,),
                    pre + "ln2.scale": (E,), pre + "ln2.bias": (E,), pre + "ffn1.kernel": (E, Md),
                    pre + "ffn1.bias": (Md,), pre + "ffn2.kernel": (Md, E), pre + "ffn2.bias": (E,)})
    out.update({"post_ln.scale": (E,), "post_ln.bias": (E,), "post.kernel": (E, Md), "post.bias": (Md,)})
    for k in range(num_mlp_layers):
        pre = f"k{k}.res."
        out.update({pre + "ln_a.scale": (Md,), pre + "ln_a.bias": (Md,), pre + "a.kernel": (Md, Md),
                    pre + "a.bias": (Md,), pre + "ln_b.scale": (Md,), pre + "ln_b.bias": (Md,),
                    pre + "b.kernel": (Md, Md), pre + "b.bias": (Md,)})
    kc = mdn_components
    out.update({"out_ln.scale": (Md,), "out_ln.bias": (Md,), "mdn.mu.kernel": (Md, kc * C), "mdn.mu.bias": (kc * C,),
                "mdn.log_sigma.kernel": (Md, kc * C), "mdn.log_sigma.bias": (kc * C,), "mdn.pi.kernel": (Md, kc),
                "mdn.pi.bias": (kc,)})
    return out


def arena_floats(shapes) -> int:
    """Each tensor starts 8-float aligned (smd_api.cu add_tensor)."""
    return sum((math.prod(s) + 7) // 8 * 8 for s in shapes.values())
