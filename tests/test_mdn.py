"""TransformerMDN on the CPU: the mixture NLL restatement against scipy, its closed-form gradient against autograd,
causality of the restated trunk, shift_right, and the plan's parameter layout (plan creation needs no GPU)."""
import math

import numpy as np
import pytest
import torch
from scipy.special import logsumexp, log_softmax
from scipy.stats import norm

from tests import mdn_reference as R


def _head(rows, kc, C, seed, ls_range=(-3.0, 2.0)):
    g = torch.Generator().manual_seed(seed)
    pi = torch.randn(rows, kc, generator=g, dtype=torch.float64) * 3
    mu = torch.randn(rows, kc * C, generator=g, dtype=torch.float64)
    ls = torch.rand(rows, kc * C, generator=g, dtype=torch.float64) * (ls_range[1] - ls_range[0]) + ls_range[0]
    x = torch.randn(rows, C, generator=g, dtype=torch.float64)
    return pi, mu, ls, x


@pytest.mark.parametrize("ls_range", [(-4.0, -2.0), (-1.0, 1.0), (1.5, 3.0)])
def test_nll_matches_scipy(ls_range):
    rows, kc, C = 7, 5, 3
    pi, mu, ls, x = _head(rows, kc, C, 0, ls_range)
    got = R.mdn_nll(pi, mu, ls, x).numpy()
    p, m, s, xx = (t.numpy() for t in (pi, mu, ls, x))
    comp = norm.logpdf(xx[:, None, :], m.reshape(rows, kc, C), np.exp(s.reshape(rows, kc, C))).sum(-1)
    ref = -logsumexp(log_softmax(p, axis=-1) + comp, axis=-1)
    np.testing.assert_allclose(got, ref, rtol=1e-12, atol=1e-10)


def test_closed_form_gradients_match_autograd():
    pi, mu, ls, x = _head(6, 4, 3, 1)
    for t in (pi, mu, ls):
        t.requires_grad_(True)
    R.mdn_nll(pi, mu, ls, x).sum().backward()
    dpi, dmu, dls = R.mdn_nll_grads(pi.detach(), mu.detach(), ls.detach(), x)
    torch.testing.assert_close(dpi, pi.grad, rtol=1e-10, atol=1e-12)
    torch.testing.assert_close(dmu, mu.grad, rtol=1e-10, atol=1e-12)
    torch.testing.assert_close(dls, ls.grad, rtol=1e-10, atol=1e-12)


def _params(C, L, Md, K, kc, seed=0):
    g = torch.Generator().manual_seed(seed)
    out = {}
    for name, shape in R.param_shapes(C, L, Md, K, kc).items():
        if name.endswith(".kernel"):
            out[name] = torch.randn(*shape, generator=g, dtype=torch.float64) / math.sqrt(shape[0])
        elif name.endswith(".scale"):
            out[name] = 1 + 0.1 * torch.randn(*shape, generator=g, dtype=torch.float64)
        else:
            out[name] = 0.1 * torch.randn(*shape, generator=g, dtype=torch.float64)
    return out


def test_oracle_attention_is_causal():
    kw = dict(num_layers=2, num_heads=8, num_mlp_layers=1, mlp_dims=64, mdn_components=3)
    p = _params(4, 2, 64, 1, 3)
    x = torch.randn(2, 32, 4, generator=torch.Generator().manual_seed(3), dtype=torch.float64)
    for shift in (False, True):
        base = R.transformer_mdn(p, x, shift=shift, **kw)
        for j in (0, 10, 31):
            x2 = x.clone()
            x2[:, j] += 1.0
            out = R.transformer_mdn(p, x2, shift=shift, **kw)
            last = j + 1 if shift else j   # outputs at positions < this see no change
            for a, b in zip(base, out):
                assert torch.equal(a[:, :last], b[:, :last])
                if last < 32:
                    assert not torch.allclose(a[:, last:], b[:, last:])


def test_shift_right():
    x = torch.arange(2 * 4 * 3, dtype=torch.float32).reshape(2, 4, 3)
    y = R.shift_right(x)
    assert torch.equal(y[:, 0], torch.zeros(2, 3)) and torch.equal(y[:, 1:], x[:, :-1])


def test_plan_layout_and_arena_size(lib):
    from smd_b200 import Engine, ModelConfig
    cfg = ModelConfig(arch="TransformerMDN", num_layers=6, num_heads=8, num_mlp_layers=2, mlp_dims=2048, channels=42,
                      mdn_components=100)
    eng = Engine(cfg, max_batch=128, training=True)
    shapes = R.param_shapes(42, 6, 2048, 2, 100)
    assert [(n, s) for n, _, s in eng.layout] == list(shapes.items())
    # the last tensor (mdn.pi.bias) ends at 38,050,484 floats; the arena rounds it up to the 8-float tensor alignment
    name, off, shape = eng.layout[-1]
    assert off + math.prod(shape) == 38_050_484
    assert eng.arena_floats == R.arena_floats(shapes) == 38_050_488
    first = eng.layout[0][1]
    assert first == 0 and not any(".film." in n for n, _, _ in eng.layout)


def test_plan_creation_rejects_unsupported_configurations(lib):
    import ctypes
    from smd_b200 import Engine, ModelConfig, lib as L
    base = dict(arch="TransformerMDN", num_layers=1, mlp_dims=256, channels=8, mdn_components=4)
    for over, kw in ((dict(seq_len=64), {}), (dict(seq_len=128), {}), (dict(mdn_components=0), {}),
                     ({}, dict(precision="bf16x3"))):
        with pytest.raises(ValueError):
            Engine(ModelConfig(**dict(base, **over)), max_batch=2, **kw)
    # the generic creation call names the right one
    c = L.SmdConfig(3, 1, 8, 2, 256, 32, 8, 2, 1, 0, 0, 0)
    h = ctypes.c_void_p()
    assert lib.smd_plan_create(ctypes.byref(c), ctypes.byref(h)) == -1
    assert b"smd_mdn_plan_create" in lib.smd_last_error()
