"""The float64 backward restatements of tests/backward_reference.py against torch.autograd through the forward
functions of oracle/ddpm_oracle.py.  The GPU stage tests compare kernels with these restatements; here the
restatements themselves are pinned, so that a wrong one cannot agree with a wrong kernel unnoticed."""
import math

import pytest
import torch

from oracle import ddpm_oracle as O
from tests import backward_reference as R

F64 = torch.float64
TOL = 1e-10


def _rand(gen, *shape, scale=1.0):
    return torch.randn(*shape, generator=gen, dtype=F64) * scale


def _close(got, want, what):
    err = float((got - want).norm() / (want.norm() + 1e-300))
    assert err < TOL, (what, err)


def _leaf(t):
    return t.clone().requires_grad_(True)


def test_bf16_round_and_ulp():
    x = torch.tensor([1.0, 1.00390625, 1.005, -3.3, 0.1, 255.0, 256.0, 1e-3, 0.0], dtype=F64)
    r = R.bf16_round(x)
    assert torch.equal(r, x.float().bfloat16().double())
    assert float(r[1]) == 1.0                         # tie: to the even significand
    u = R.bf16_ulp(x)
    assert float(u[0]) == 2.0 ** -7 and float(u[3]) == 2.0 ** -6 and float(u[5]) == 1.0 and float(u[6]) == 2.0
    nz = x != 0
    assert bool(((r - x).abs()[nz] <= 0.5 * u[nz]).all())
    nxt = (r + u * torch.sign(r))[nz]                 # one spacing further out is again a bfloat16 number
    assert torch.equal(R.bf16_round(nxt), nxt)


def test_dense_adjoints():
    g = torch.Generator().manual_seed(1)
    x, w, b = _leaf(_rand(g, 3, 5, 7)), _leaf(_rand(g, 7, 4)), _leaf(_rand(g, 4))
    dy = _rand(g, 3, 5, 4)
    (O.dense(x, w, b) * dy).sum().backward()
    _close(R.dense_bwd_w(x.detach(), dy), w.grad, "dW")
    _close(R.dense_bwd_x(dy, w.detach()), x.grad, "dx")
    _close(R.dense_bwd_b(dy), b.grad, "db")


def test_activation_derivatives():
    x = _leaf(torch.linspace(-9.0, 9.0, 1801, dtype=F64))
    O.gelu_tanh(x).sum().backward()
    _close(R.gelu_tanh_grad(x.detach()), x.grad, "gelu'")
    # the tanh form is not the erf form: the two derivatives differ by up to ~1e-3, which the stage rules resolve
    xd = x.detach()
    erf_grad = 0.5 * (1 + torch.erf(xd / math.sqrt(2))) + xd * torch.exp(-0.5 * xd * xd) / math.sqrt(2 * math.pi)
    assert 1e-4 < float((R.gelu_tanh_grad(xd) - erf_grad).abs().max()) < 1e-2
    x.grad = None
    O.swish(x).sum().backward()
    _close(R.swish_grad(x.detach()), x.grad, "swish'")


@pytest.mark.parametrize("n", [128, 2048])
def test_layer_norm_with_residual(n):
    """The 128-wide LayerNorms of the trunk: out = f(LayerNorm(h)) + h, so dh = LayerNorm adjoint + residual adjoint."""
    g = torch.Generator().manual_seed(2)
    h = _leaf(_rand(g, 2, 6, n) * 1.7 + 0.3)
    gamma, beta = _leaf(1 + _rand(g, n, scale=0.1)), _leaf(_rand(g, n, scale=0.1))
    dy, dres = _rand(g, 2, 6, n), _rand(g, 2, 6, n)
    ((O.layer_norm(h, gamma, beta) * dy).sum() + (h * dres).sum()).backward()
    dx, dgamma, dbeta = R.layer_norm_bwd(dy, h.detach(), gamma.detach())
    _close(dx + dres, h.grad, "dh")
    _close(dgamma, gamma.grad, "dgamma")
    _close(dbeta, beta.grad, "dbeta")
    dx2, _, _ = R.layer_norm_bwd(dy, h.detach(), gamma.detach(), R.row_stats(h.detach()))
    assert torch.equal(dx, dx2)


@pytest.mark.parametrize("rows_per_example", [1, 32])
def test_layer_norm_film_swish(rows_per_example):
    """Both uses of a FiLM pair inside a DenseResBlock (models/shared.py:62-68): the pair's adjoint is the sum."""
    g = torch.Generator().manual_seed(3)
    B, S, N = 3, rows_per_example, 256
    x = _leaf(_rand(g, B, S, N) * 2.0 - 0.5)
    gamma, beta = _leaf(1 + _rand(g, N, scale=0.1)), _leaf(_rand(g, N, scale=0.1))
    scale, shift = _leaf(1 + _rand(g, B, N, scale=0.3)), _leaf(_rand(g, B, N, scale=0.3))
    dy = _rand(g, B, S, N)
    out = O.swish(scale[:, None, :] * O.layer_norm(x, gamma, beta) + shift[:, None, :])
    (out * dy).sum().backward()
    dx, dgamma, dbeta, dscale, dshift = R.ln_film_swish_bwd(dy, x.detach(), gamma.detach(), beta.detach(),
                                                            scale.detach(), shift.detach(), R.row_stats(x.detach()))
    for got, want, what in ((dx, x.grad, "dx"), (dgamma, gamma.grad, "dgamma"), (dbeta, beta.grad, "dbeta"),
                            (dscale, scale.grad, "dscale"), (dshift, shift.grad, "dshift")):
        _close(got, want, what)


def test_dense_res_block_chain():
    """The stage rules chain ln_b, dense a, ln_a and the skip connection exactly like this."""
    g = torch.Generator().manual_seed(4)
    B, S, N = 2, 4, 64
    names = ["ln_a.scale", "ln_a.bias", "a.kernel", "a.bias", "ln_b.scale", "ln_b.bias", "b.kernel", "b.bias"]
    p = {}
    for nm in names:
        base = _rand(g, N, N, scale=N ** -0.5) if nm.endswith("kernel") else _rand(g, N, scale=0.1)
        p["r." + nm] = _leaf(base + (1.0 if nm.endswith("scale") else 0.0))
    x = _leaf(_rand(g, B, S, N))
    scale, shift = _leaf(1 + _rand(g, B, N, scale=0.3)), _leaf(_rand(g, B, N, scale=0.3))
    dy = _rand(g, B, S, N)
    (O.dense_res_block(x, scale[:, None, :], shift[:, None, :], p, "r.") * dy).sum().backward()
    d = {k: v.detach() for k, v in p.items()}
    with torch.no_grad():
        act_a = O.swish(scale[:, None] * O.layer_norm(x, d["r.ln_a.scale"], d["r.ln_a.bias"]) + shift[:, None])
        r1 = O.dense(act_a, d["r.a.kernel"], d["r.a.bias"])
        act_b = O.swish(scale[:, None] * O.layer_norm(r1, d["r.ln_b.scale"], d["r.ln_b.bias"]) + shift[:, None])
    _close(R.dense_bwd_w(act_b, dy), p["r.b.kernel"].grad, "dWb")
    _close(R.dense_bwd_b(dy), p["r.b.bias"].grad, "dbb")
    dr1, dg_b, db_b, dsc_b, dsh_b = R.ln_film_swish_bwd(R.dense_bwd_x(dy, d["r.b.kernel"]), r1, d["r.ln_b.scale"],
                                                        d["r.ln_b.bias"], scale.detach(), shift.detach())
    _close(R.dense_bwd_w(act_a, dr1), p["r.a.kernel"].grad, "dWa")
    _close(R.dense_bwd_b(dr1), p["r.a.bias"].grad, "dba")
    dx, dg_a, db_a, dsc_a, dsh_a = R.ln_film_swish_bwd(R.dense_bwd_x(dr1, d["r.a.kernel"]), x.detach(),
                                                       d["r.ln_a.scale"], d["r.ln_a.bias"], scale.detach(),
                                                       shift.detach())
    _close(dx + dy, x.grad, "dx")
    _close(dg_b, p["r.ln_b.scale"].grad, "dgamma_b")
    _close(db_a, p["r.ln_a.bias"].grad, "dbeta_a")
    _close(dsc_a + dsc_b, scale.grad, "dscale")
    _close(dsh_a + dsh_b, shift.grad, "dshift")


@pytest.mark.parametrize("S", [32, 64, 128])
@pytest.mark.parametrize("H", [4, 8, 16, 32])
@pytest.mark.parametrize("causal", [False, True])
def test_attention(H, S, causal):
    g = torch.Generator().manual_seed(100 * H + S)
    B, E = 2, 128
    qkv = _leaf(_rand(g, B, S, 3 * E))
    d_out = _rand(g, B, S, E)
    # O.self_attention with a zero input, qkv as a full-shape "bias" and an identity output projection is the bare
    # attention core on qkv
    p = {"a.qkv.kernel": torch.zeros(E, 3 * E, dtype=F64), "a.qkv.bias": qkv,
         "a.out.kernel": torch.eye(E, dtype=F64), "a.out.bias": torch.zeros(E, dtype=F64)}
    x = torch.zeros(B, S, E, dtype=F64)
    if causal:
        from tests import mdn_reference as MR
        out = MR.self_attention(x, p, "a.", H, causal=True)
    else:
        out = O.self_attention(x, p, "a.", H)
    (out * d_out).sum().backward()
    with torch.no_grad():
        dh = E // H
        q, k, _ = (t.reshape(B, S, H, dh) for t in qkv.detach().split(E, dim=-1))
        logits = torch.einsum("bqhd,bkhd->bhqk", q, k) / math.sqrt(dh)
        if causal:
            logits = logits.masked_fill(torch.ones(S, S).triu(1).bool(), float("-inf"))
        probs = torch.softmax(logits, dim=-1)
    _close(R.attention_bwd(qkv.detach(), probs, d_out, H), qkv.grad, "dqkv")


def test_film_generator():
    g = torch.Generator().manual_seed(5)
    B, N = 5, 96
    p = {"f.d1.kernel": _rand(g, 128, 512, scale=128 ** -0.5), "f.d1.bias": _rand(g, 512, scale=0.1),
         "f.d2.kernel": _rand(g, 512, 512, scale=512 ** -0.5), "f.d2.bias": _rand(g, 512, scale=0.1),
         "f.ss.kernel": _rand(g, 512, 2 * N, scale=512 ** -0.5), "f.ss.bias": _rand(g, 2 * N, scale=0.1)}
    p = {k: _leaf(v) for k, v in p.items()}
    t = torch.rand(B, generator=g, dtype=F64)
    dss = _rand(g, B, 2 * N)
    scale, shift = O.dense_film(t, p, "f.")
    (torch.cat([scale, shift], dim=-1) * dss).sum().backward()
    with torch.no_grad():
        enc = O.noise_encoding(t, 128)
        e1pre = O.dense(enc, p["f.d1.kernel"], p["f.d1.bias"])
        e1 = O.swish(e1pre)
        e2 = O.dense(e1, p["f.d2.kernel"], p["f.d2.bias"])
    got = R.film_generator_bwd(dss, enc, e1pre, e1, e2, p["f.ss.kernel"].detach(), p["f.d2.kernel"].detach())
    for name in ("ss.kernel", "ss.bias", "d2.kernel", "d2.bias", "d1.kernel", "d1.bias"):
        _close(got[name], p["f." + name].grad, name)


@pytest.mark.parametrize("shape", [(3, 32, 42), (4, 512)])
def test_loss_seeds(shape):
    g = torch.Generator().manual_seed(6)
    B, global_batch = shape[0], 2 * shape[0]
    x0, eps = _rand(g, *shape), _rand(g, *shape)
    # ddpm: O.diffusion_loss_tensors(reduction="sum") / global_batch is this shard's part of the global mean
    pred = _leaf(_rand(g, *shape))
    used = torch.rand(B, generator=g, dtype=F64) * 0.9 + 0.05
    loss, _ = O.diffusion_loss_tensors(lambda x, t: pred, x0, used, eps, "none")
    (loss.sum() / global_batch).backward()
    got_loss, dpred = R.ddpm_loss_seed(eps, pred.detach(), global_batch)
    _close(got_loss, loss.detach(), "ddpm loss")
    _close(dpred, pred.grad, "ddpm dpred")
    # dsm: the network's score is raw / sigma
    raw = _leaf(_rand(g, *shape))
    sig = torch.rand(B, generator=g, dtype=F64) + 0.1
    loss, _ = O.dsm_loss_tensors(lambda x, s: raw / s, x0, sig, eps, "none")
    (loss.sum() / global_batch).backward()
    got_loss, draw = R.dsm_loss_seed(eps, raw.detach(), global_batch)
    _close(got_loss, loss.detach(), "dsm loss")
    _close(draw, raw.grad, "dsm draw")
