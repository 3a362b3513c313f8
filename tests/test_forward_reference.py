"""The float64 forward restatements of tests/forward_reference.py against the networks of oracle/ddpm_oracle.py.

tests/test_gpu_forward_stages.py compares every forward launch with one of these restatements; here the restatements,
composed launch by launch in the order the forward pass runs them, must reproduce the oracle's TransformerDDPM,
DenseDDPM and DenseNCSN to 1e-12, so that a wrong restatement cannot agree with a wrong kernel unnoticed."""
import math

import pytest
import torch

from oracle import ddpm_oracle as O
from tests import forward_reference as F

F64 = torch.float64
TOL = 1e-12


def _close(got, want, what, tol=TOL):
    err = float((got - want).norm() / (want.norm() + 1e-300))
    assert err < tol, (what, err)


def _params(seed, C, Md, L, K, dense):
    """A random parameter dict under the workspace names, LayerNorm and bias terms perturbed away from 1 / 0."""
    g = torch.Generator().manual_seed(seed)
    p = {}

    def lin(name, i, o):
        p[name + ".kernel"] = torch.randn(i, o, generator=g, dtype=F64) / math.sqrt(i)
        p[name + ".bias"] = 0.1 * torch.randn(o, generator=g, dtype=F64)

    def norm(name, n):
        p[name + ".scale"] = 1.0 + 0.1 * torch.randn(n, generator=g, dtype=F64)
        p[name + ".bias"] = 0.1 * torch.randn(n, generator=g, dtype=F64)

    if dense:
        lin("in", C, Md)
    else:
        lin("in", C, 128)
        for l in range(L):
            norm(f"l{l}.ln1", 128)
            lin(f"l{l}.attn.qkv", 128, 384)
            lin(f"l{l}.attn.out", 128, 128)
            norm(f"l{l}.ln2", 128)
            lin(f"l{l}.ffn1", 128, Md)
            lin(f"l{l}.ffn2", Md, 128)
        norm("post_ln", 128)
        lin("post", 128, Md)
    for k in range(K):
        lin(f"k{k}.film.d1", 128, 512)
        lin(f"k{k}.film.d2", 512, 512)
        lin(f"k{k}.film.ss", 512, 2 * Md)
        norm(f"k{k}.res.ln_a", Md)
        lin(f"k{k}.res.a", Md, Md)
        norm(f"k{k}.res.ln_b", Md)
        lin(f"k{k}.res.b", Md, Md)
    norm("out_ln", Md)
    lin("out", Md, C)
    return p


def _sub(p, pre):
    return {k[len(pre):]: v for k, v in p.items() if k.startswith(pre)}


FREQS = O._sinusoid_freqs(64, F64)


def _tail(p, u, t, B, S, K, broadcast):
    """post / in GEMM output u (M, Md) -> network output, launch by launch as run_tail runs them."""
    M = u.shape[0]
    for k in range(K):
        ss = F.film_generator(t[:1] if broadcast else t, FREQS, _sub(p, f"k{k}.film."), arg32=False)["ss"]
        rows = F.film_rows(ss, M, S, broadcast=broadcast)
        pre = f"k{k}.res."
        acta, _ = F.ln_film_act(u, F.row_stats(u), p[pre + "ln_a.scale"], p[pre + "ln_a.bias"], rows, True)
        r1 = F.gemm(acta, p[pre + "a.kernel"], p[pre + "a.bias"])
        actb, _ = F.ln_film_act(r1["v"], r1["stats"], p[pre + "ln_b.scale"], p[pre + "ln_b.bias"], rows, True)
        u = F.gemm(actb, p[pre + "b.kernel"], p[pre + "b.bias"], residual=u)["v"]
    act_out, _ = F.ln_film_act(u, F.row_stats(u), p["out_ln.scale"], p["out_ln.bias"], None, False)
    return F.gemm(act_out, p["out.kernel"], p["out.bias"])["v"]


def _transformer(p, x, t, L, K, H, fused, broadcast=False):
    B, S, C = x.shape
    h, a = F.embed(x.reshape(B, S, C), p["in.kernel"], p["in.bias"], O.transformer_positional_encoding(S, 128, F64),
                   p["l0.ln1.scale"], p["l0.ln1.bias"])
    h, a = h.reshape(B * S, 128), a.reshape(B * S, 128)
    for l in range(L):
        pre = f"l{l}."
        nxt = f"l{l + 1}.ln1." if l + 1 < L else "post_ln."
        ln2 = (p[pre + "ln2.scale"], p[pre + "ln2.bias"])
        if fused:
            h, a2 = F.attn_block(a.reshape(B, S, 128), h.reshape(B, S, 128), p[pre + "attn.qkv.kernel"],
                                 p[pre + "attn.qkv.bias"], p[pre + "attn.out.kernel"], p[pre + "attn.out.bias"], *ln2,
                                 H, round_o=False)
            h, a2 = h.reshape(B * S, 128), a2.reshape(B * S, 128)
            h, a = F.ffn_fused(a2, h, p[pre + "ffn1.kernel"], p[pre + "ffn1.bias"], p[pre + "ffn2.kernel"],
                               p[pre + "ffn2.bias"], p[nxt + "scale"], p[nxt + "bias"], round_hidden=False)
            continue
        qkv = F.gemm(a, p[pre + "attn.qkv.kernel"], p[pre + "attn.qkv.bias"])["v"]
        _, o = F.attention(qkv.reshape(B, S, 384), H)
        e = F.gemm(o.reshape(B * S, 128), p[pre + "attn.out.kernel"], p[pre + "attn.out.bias"], residual=h, ln=ln2)
        h, a2 = e["v"], e["ln"]
        hid = F.gemm(a2, p[pre + "ffn1.kernel"], p[pre + "ffn1.bias"], act="gelu")["act"]
        e = F.gemm(hid, p[pre + "ffn2.kernel"], p[pre + "ffn2.bias"], residual=h, ln=(p[nxt + "scale"], p[nxt + "bias"]))
        h, a = e["v"], e["ln"]
    u = F.gemm(a, p["post.kernel"], p["post.bias"])["v"]
    return _tail(p, u, t, B, S, K, broadcast).reshape(B, S, C)


@pytest.mark.parametrize("S,H,C,fused", [(32, 8, 42, False), (32, 8, 42, True), (64, 16, 42, True),
                                         (128, 16, 42, False), (32, 4, 42, False), (32, 32, 146, False)])
def test_transformer_composition_is_the_oracle(S, H, C, fused):
    L, K, Md, B = 2, 2, 256, 3
    p = _params(S + H + C, C, Md, L, K, dense=False)
    g = torch.Generator().manual_seed(7)
    x = torch.rand(B, S, C, generator=g, dtype=F64) * 2 - 1
    t = torch.rand(B, generator=g, dtype=F64) * 0.9 + 0.05
    ref = O.transformer_ddpm(p, x, t, num_layers=L, num_heads=H, num_mlp_layers=K, mlp_dims=Md)
    _close(_transformer(p, x, t, L, K, H, fused), ref, f"S{S} H{H} C{C} fused={fused}")


def test_transformer_broadcast_t_is_the_oracle_with_t_repeated():
    L, K, Md, B, S, C, H = 1, 2, 256, 3, 32, 42, 8
    p = _params(3, C, Md, L, K, dense=False)
    g = torch.Generator().manual_seed(8)
    x = torch.rand(B, S, C, generator=g, dtype=F64) * 2 - 1
    t = torch.full((B,), 0.37, dtype=F64)
    ref = O.transformer_ddpm(p, x, t, num_layers=L, num_heads=H, num_mlp_layers=K, mlp_dims=Md)
    _close(_transformer(p, x, t[:1], L, K, H, fused=False, broadcast=True), ref, "broadcast t")


@pytest.mark.parametrize("arch", ["DenseDDPM", "DenseNCSN"])
def test_dense_composition_is_the_oracle(arch):
    K, C, Md, B = 2, 64, 256, 5
    p = _params(11, C, Md, 0, K, dense=True)
    g = torch.Generator().manual_seed(9)
    x = torch.rand(B, C, generator=g, dtype=F64) * 2 - 1
    t = torch.rand(B, generator=g, dtype=F64) * 0.9 + 0.05
    u = F.gemm(x, p["in.kernel"], p["in.bias"])["v"]
    y = _tail(p, u, t, B, 1, K, False)
    if arch == "DenseNCSN":
        _close(F.scale_rows(y, t), O.dense_ncsn(p, x, t, num_layers=K, mlp_dims=Md), arch)
    else:
        _close(y, O.dense_ddpm(p, x, t, num_layers=K, mlp_dims=Md), arch)


def test_explicit_film_row_selects_that_row_for_every_token():
    g = torch.Generator().manual_seed(4)
    ss = torch.randn(5, 8, generator=g, dtype=F64)
    assert torch.equal(F.film_rows(ss, 7, 1, row=3), ss[3].expand(7, -1))
    assert torch.equal(F.film_rows(ss, 64, 32), torch.cat([ss[0].expand(32, -1), ss[1].expand(32, -1)]))
    assert torch.equal(F.film_rows(ss, 3, 32, broadcast=True), ss[0].expand(3, -1))


@pytest.mark.parametrize("H,S", [(8, 32), (16, 64)])
def test_fused_attention_block_without_rounding_is_the_unfused_composition(H, S):
    g = torch.Generator().manual_seed(5)
    p = _params(5, 42, 256, 1, 0, dense=False)
    a, h = torch.randn(2, S, 128, generator=g, dtype=F64), torch.randn(2, S, 128, generator=g, dtype=F64)
    args = (p["l0.attn.qkv.kernel"], p["l0.attn.qkv.bias"], p["l0.attn.out.kernel"], p["l0.attn.out.bias"],
            p["l0.ln2.scale"], p["l0.ln2.bias"], H)
    h_mid, a2 = F.attn_block(a, h, *args, round_o=False)
    _, o = F.attention(F.gemm(a, args[0], args[1])["v"], H)
    e = F.gemm(o, args[2], args[3], residual=h, ln=(args[4], args[5]))
    _close(h_mid, e["v"], "h_mid")
    _close(a2, e["ln"], "a2")
    _close(a2, O.layer_norm(h + O.self_attention(a, _sub(p, "l0."), "attn.", H), args[4], args[5]), "oracle")
    h_r, _ = F.attn_block(a, h, *args, round_o=True)     # rounding o is a change of the size of one bf16 rounding
    assert 1e-5 < float((h_r - h_mid).norm() / h_mid.norm()) < 1e-2


def test_fused_ffn_without_rounding_is_the_unfused_composition():
    g = torch.Generator().manual_seed(6)
    p = _params(6, 42, 512, 1, 0, dense=False)
    a2, h = torch.randn(70, 128, generator=g, dtype=F64), torch.randn(70, 128, generator=g, dtype=F64)
    args = (p["l0.ffn1.kernel"], p["l0.ffn1.bias"], p["l0.ffn2.kernel"], p["l0.ffn2.bias"], p["post_ln.scale"],
            p["post_ln.bias"])
    h_out, a_next = F.ffn_fused(a2, h, *args, round_hidden=False)
    up = F.gemm(a2, args[0], args[1], act="gelu")
    e = F.gemm(up["act"], args[2], args[3], residual=h, ln=(args[4], args[5]))
    _close(h_out, e["v"], "h_out")
    _close(a_next, e["ln"], "a_next")
    _close(up["act"], O.gelu_tanh(up["v"]), "gelu")
    h_r, _ = F.ffn_fused(a2, h, *args, round_hidden=True)
    assert 1e-5 < float((h_r - h_out).norm() / h_out.norm()) < 1e-2


def test_causal_attention_zeroes_the_upper_triangle_and_matches_masked_softmax():
    g = torch.Generator().manual_seed(7)
    qkv = torch.randn(2, 32, 384, generator=g, dtype=F64)
    probs, o = F.attention(qkv, 8, causal=True)
    assert bool((probs * torch.ones(32, 32, dtype=F64).triu(1) == 0).all())
    _close(probs.sum(-1), torch.ones_like(probs.sum(-1)), "rows sum to 1")
    # flax's causal mask: a -1e10 bias above the diagonal
    q, k, v = (t.reshape(2, 32, 8, 16) for t in qkv.split(128, dim=-1))
    logits = torch.einsum("bqhd,bkhd->bhqk", q / 4.0, k) - 1e10 * torch.ones(32, 32, dtype=F64).triu(1)
    _close(o, torch.einsum("bhqk,bkhd->bqhd", torch.softmax(logits, -1), v).reshape(2, 32, 128), "o")


@pytest.mark.parametrize("film,act", [(True, True), (False, False), (True, False)])
def test_tangent_is_the_jvp_of_layer_norm_film_swish(film, act):
    g = torch.Generator().manual_seed(8)
    M, N = 6, 256
    x = torch.randn(M, N, generator=g, dtype=F64) * 1.3 + 0.2
    xt = torch.randn(M, N, generator=g, dtype=F64)
    gamma, beta = 1 + 0.1 * torch.randn(N, generator=g, dtype=F64), 0.1 * torch.randn(N, generator=g, dtype=F64)
    rows = torch.randn(M, 2 * N, generator=g, dtype=F64) if film else None

    def fwd(xx):
        y = O.layer_norm(xx, gamma, beta)
        if film:
            y = rows[:, :N] * y + rows[:, N:]
        return O.swish(y) if act else y

    _, want = torch.autograd.functional.jvp(fwd, x, xt)
    _close(F.ln_film_tangent(x, F.row_stats(x), xt, gamma, beta, rows, act), want, "tangent")
    out, z = F.ln_film_act(x, None, gamma, beta, rows, act)
    _close(out, fwd(x), "primal")


def test_noise_encoding_argument_is_rounded_as_float32_products():
    t = torch.tensor([0.05, 0.3711, 0.999], dtype=F64)
    f32 = O._sinusoid_freqs(64, torch.float32)
    arg = F.noise_arg_f32(t, f32.to(F64))
    want = (5000 * t.float())[:, None] * f32[None, :]
    assert torch.equal(arg, want.to(F64))
    _close(F.noise_encoding(t, FREQS), O.noise_encoding(t, 128), "fp64 noise encoding")


def test_activation_excess_is_zero_for_a_rounded_exact_value_and_measures_the_rest():
    v = torch.linspace(-12, 6, 10001, dtype=F64)
    ref = F.swish(v)
    assert float(F.activation_excess(F.bf16_round(ref), ref, v).max()) == 0.0
    # an error of |v| 2^-12 on top of the rounding is measured as such (to the rounding's slack)
    got = F.bf16_round(ref + v.abs() * 2.0 ** -12)
    assert float(F.activation_excess(got, ref, v).max()) <= 2.0 ** -12 * 1.01 + 1e-300
    assert float(F.activation_excess(got, ref, v).max()) > 2.0 ** -13
