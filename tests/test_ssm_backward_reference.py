"""The float64 second-order LayerNorm backward of sliced score matching (backward_reference.ssm_ln_film_swish_bwd),
pinned four ways before tests/test_gpu_ssm_backward_stages.py compares ssm_ln_bwd_kernel with it:

- against a separate restatement of the closed form in the comment above SsmLnBwdArgs (csrc/backward_kernels.cuh),
  which checks that formula in float64;
- against central differences of the functional it differentiates;
- against the first-order backward (g' = 0) and against the plain LayerNorm (no FiLM, no activation);
- chained launch by launch over a float64 DenseNCSN, against the reverse-over-reverse parameter gradients of
  ssm_reference.ssm_loss_tensors: the launch decomposition the GPU rules assume is the right one.

A sensitivity test shows that the GPU bounds would notice a kernel that drops any single term of the closed form."""

import pytest
import torch

from oracle import ddpm_oracle as O
from tests import backward_reference as R
from tests import forward_reference as F
from tests import ssm_reference as SR

F64 = torch.float64
SIGMAS = O.create_noise_schedule(1.0, 0.01, 15, "geometric")
TERMS = ("swish2", "q", "gr", "gP", "dscale_t")


def _rel(got, want):
    return float((got - want).norm() / (want.norm() + 1e-300))


def _rand(gen, *shape, scale=1.0, shift=0.0):
    return torch.randn(*shape, generator=gen, dtype=F64) * scale + shift


def closed_form(g, gt, x, xt, gamma, beta, scale, shift, stats, act, drop=()):
    """The formula of the comment above SsmLnBwdArgs, term by term; `drop` removes the named terms (TERMS)."""
    n = x.shape[-1]
    mean = (stats[..., 0] / n).unsqueeze(-1)
    r = torch.rsqrt(stats[..., 1].unsqueeze(-1) / n - mean * mean + R.LN_EPS)
    xh = (x - mean) * r
    xc = xt - xt.mean(dim=-1, keepdim=True)
    m2 = (xh * xt).mean(dim=-1, keepdim=True)
    q = r * m2
    xhd = r * xc - xh * q
    y, yd = gamma * xh + beta, gamma * xhd
    s = scale[:, None, :] if scale is not None else torch.ones_like(gamma)
    h = shift[:, None, :] if scale is not None else torch.zeros_like(gamma)
    z, zd = s * y + h, s * yd
    if act == "swish":
        sg = torch.sigmoid(z)
        d1 = sg * (1 + z * (1 - sg))
        d2 = sg * (1 - sg) * (2 + z * (1 - 2 * sg))
        gz = g * d1 + (0 if "swish2" in drop else gt * d2 * zd)
        gzd = gt * d1
    else:
        gz, gzd = g, gt
    dscale = (gz * y + (0 if "dscale_t" in drop else gzd * yd)).sum(dim=1)
    dshift = gz.sum(dim=1)
    gxh, gxd = gz * s * gamma, gzd * s * gamma
    hh = gxh - (0 if "q" in drop else q * gxd)
    mean_ = lambda t: t.mean(dim=-1, keepdim=True)
    sum_ = lambda t: t.sum(dim=-1, keepdim=True)
    gr = sum_(gxd * xc) - 2 * m2 * sum_(gxd * xh)
    gP = -r * r * sum_(gxd * xh)
    dx = r * (hh - mean_(hh) - xh * mean_(xh * hh))
    if "gr" not in drop:
        dx = dx - r * r * xh / n * gr
    if "gP" not in drop:
        dx = dx + xc / n * gP
    dxt = r * (gxd - mean_(gxd) - xh * mean_(xh * gxd))
    flat = lambda t: t.reshape(-1, n).sum(dim=0)
    dgamma = flat(gz * s * xh + gzd * s * xhd)
    dbeta = flat(gz * s)
    return dx, dxt, dgamma, dbeta, (dscale if scale is not None else None), (dshift if scale is not None else None)


def _case(seed, B=3, S=2, N=96, film=True):
    gen = torch.Generator().manual_seed(seed)
    x = _rand(gen, B, S, N, scale=1.3, shift=0.4)
    return dict(g=_rand(gen, B, S, N), gt=_rand(gen, B, S, N, scale=0.7), x=x, xt=_rand(gen, B, S, N),
                gamma=_rand(gen, N, scale=0.2, shift=1.0), beta=_rand(gen, N, scale=0.2),
                scale=_rand(gen, B, N, scale=0.3, shift=1.0) if film else None,
                shift=_rand(gen, B, N, scale=0.5) if film else None, stats=R.row_stats(x),
                act="swish" if film else None)


@pytest.mark.parametrize("film", [True, False])
def test_autograd_reference_equals_the_kernel_closed_form(film):
    a = _case(1, film=film)
    got = R.ssm_ln_film_swish_bwd(**a)
    want = closed_form(**a)
    for name, gv, wv in zip(("dx", "dxt", "dgamma", "dbeta", "dscale", "dshift"), got, want):
        if wv is None:
            assert gv is None, name
            continue
        err = _rel(gv, wv)
        assert err < 1e-12, (name, err)


def _functional(g, gt, x, xt, gamma, beta, scale, shift, act):
    """<g, out> + <g', out'> with the statistics of x itself; out' from forward_reference's tangent formula."""
    B, S, N = x.shape
    rows = None if scale is None else torch.cat([scale, shift], dim=-1).repeat_interleave(S, dim=0)
    xf, xtf = x.reshape(B * S, N), xt.reshape(B * S, N)
    st = R.row_stats(xf)
    out, _ = F.ln_film_act(xf, st, gamma, beta, rows, act == "swish")
    out_t = F.ln_film_tangent(xf, st, xtf, gamma, beta, rows, act == "swish")
    return float((g.reshape(B * S, N) * out).sum() + (gt.reshape(B * S, N) * out_t).sum())


@pytest.mark.parametrize("film", [True, False])
def test_autograd_reference_matches_central_differences(film):
    a = _case(2, N=64, film=film)
    grads = R.ssm_ln_film_swish_bwd(**a)
    names = ("x", "xt", "gamma", "beta") + (("scale", "shift") if film else ())
    gen = torch.Generator().manual_seed(3)
    for name, grad in zip(names, grads):
        d = torch.randn(a[name].shape, generator=gen, dtype=F64)
        h = 1e-5
        kw = {k: a[k] for k in ("g", "gt", "x", "xt", "gamma", "beta", "scale", "shift", "act")}
        plus, minus = dict(kw), dict(kw)
        plus[name], minus[name] = a[name] + h * d, a[name] - h * d
        fd = (_functional(**plus) - _functional(**minus)) / (2 * h)
        an = float((grad * d).sum())
        assert abs(fd - an) <= 1e-7 * max(1.0, abs(an)), (name, fd, an)


def test_without_tangent_adjoint_it_is_the_first_order_backward():
    a = _case(4)
    a["gt"] = torch.zeros_like(a["gt"])
    dx, dxt, dgamma, dbeta, dscale, dshift = R.ssm_ln_film_swish_bwd(**a)
    want = R.ln_film_swish_bwd(a["g"], a["x"], a["gamma"], a["beta"], a["scale"], a["shift"], a["stats"])
    for name, gv, wv in zip(("dx", "dgamma", "dbeta", "dscale", "dshift"), (dx, dgamma, dbeta, dscale, dshift), want):
        assert _rel(gv, wv) < 1e-13, name
    assert bool((dxt == 0).all())


def test_plain_layer_norm_second_order_backward():
    """No FiLM, no activation: the gradient of <g, LN(x)> + <g', J_LN(x) x'> through torch.func.jvp of the oracle's
    LayerNorm, a third derivation."""
    a = _case(5, film=False)
    dx, dxt, dgamma, dbeta, dscale, dshift = R.ssm_ln_film_swish_bwd(**a)
    assert dscale is None and dshift is None
    leaves = [a[k].clone().requires_grad_(True) for k in ("x", "xt", "gamma", "beta")]
    out, out_t = torch.func.jvp(lambda u: O.layer_norm(u, leaves[2], leaves[3]), (leaves[0],), (leaves[1],))
    ((a["g"] * out).sum() + (a["gt"] * out_t).sum()).backward()
    for name, gv, leaf in zip(("dx", "dxt", "dgamma", "dbeta"), (dx, dxt, dgamma, dbeta), leaves):
        assert _rel(gv, leaf.grad) < 1e-12, name
    want_dx, want_dg, want_db = R.layer_norm_bwd(a["g"], a["x"], a["gamma"])
    a["gt"] = torch.zeros_like(a["gt"])
    dx0, _, dg0, db0, _, _ = R.ssm_ln_film_swish_bwd(**a)
    assert _rel(dx0, want_dx) < 1e-13 and _rel(dg0, want_dg) < 1e-13 and _rel(db0, want_db) < 1e-13


# ----------------------------------------------------------------------------------------------------------------------
# the launch decomposition of the sliced score matching train step, in float64
# ----------------------------------------------------------------------------------------------------------------------
def ssm_step_fp64(p, x0, sig, eps, v, K, gb):
    """One sliced score matching gradient of DenseNCSN composed from the per-launch rules of the device step
    (csrc/backward.cu ssm_grads_impl), every operand in float64.  Returns (gradients by arena name, the inputs of every
    ssm_ln_bwd launch as (kind, kwargs of ssm_ln_film_swish_bwd, the residual adjoint added to its dx or None))."""
    B, N = x0.shape[0], p["in.kernel"].shape[1]
    xt = x0 + sig[:, None] * eps
    enc = O.noise_encoding(sig, 128)
    u, ut = [xt @ p["in.kernel"] + p["in.bias"]], [v @ p["in.kernel"]]
    film, acts, r1s = [], [], []
    for k in range(K):
        fp, pre = f"k{k}.film.", f"k{k}.res."
        e1pre = enc @ p[fp + "d1.kernel"] + p[fp + "d1.bias"]
        e1 = O.swish(e1pre)
        e2 = e1 @ p[fp + "d2.kernel"] + p[fp + "d2.bias"]
        ss = e2 @ p[fp + "ss.kernel"] + p[fp + "ss.bias"]
        film.append((e1pre, e1, e2, ss))
        rows = ss
        st = R.row_stats(u[k])
        acta, _ = F.ln_film_act(u[k], st, p[pre + "ln_a.scale"], p[pre + "ln_a.bias"], rows, True)
        actta = F.ln_film_tangent(u[k], st, ut[k], p[pre + "ln_a.scale"], p[pre + "ln_a.bias"], rows, True)
        r1, r1t = acta @ p[pre + "a.kernel"] + p[pre + "a.bias"], actta @ p[pre + "a.kernel"]
        st1 = R.row_stats(r1)
        actb, _ = F.ln_film_act(r1, st1, p[pre + "ln_b.scale"], p[pre + "ln_b.bias"], rows, True)
        acttb = F.ln_film_tangent(r1, st1, r1t, p[pre + "ln_b.scale"], p[pre + "ln_b.bias"], rows, True)
        u.append(actb @ p[pre + "b.kernel"] + p[pre + "b.bias"] + u[k])
        ut.append(acttb @ p[pre + "b.kernel"] + ut[k])
        acts.append((acta, actta, actb, acttb))
        r1s.append((r1, r1t))
    stK = R.row_stats(u[K])
    act_out, _ = F.ln_film_act(u[K], stK, p["out_ln.scale"], p["out_ln.bias"], None, False)
    actt_out = F.ln_film_tangent(u[K], stK, ut[K], p["out_ln.scale"], p["out_ln.bias"], None, False)
    f = act_out @ p["out.kernel"] + p["out.bias"]
    # objective 0.5 |f|^2 + sigma v.f' per example, mean over the global batch: the two seeds
    dpred, dpredt = f / gb, sig[:, None] * v / gb
    grads, launches = {}, []
    grads["out.bias"] = R.dense_bwd_b(dpred)
    grads["out.kernel"] = R.dense_bwd_w(act_out, dpred) + R.dense_bwd_w(actt_out, dpredt)

    def ln(kind, g, gt, x, xt, pre, rows, dres=None):
        kw = dict(g=g[:, None], gt=gt[:, None], x=x[:, None], xt=xt[:, None], gamma=p[pre + "scale"],
                  beta=p[pre + "bias"], scale=None if rows is None else rows[:, :N],
                  shift=None if rows is None else rows[:, N:], stats=R.row_stats(x)[:, None],
                  act=None if rows is None else "swish")
        launches.append((kind, kw, dres))
        dx, dxt, dg, db, dsc, dsh = R.ssm_ln_film_swish_bwd(**kw)
        grads[pre + "scale"], grads[pre + "bias"] = dg, db
        return dx[:, 0], dxt[:, 0], dsc, dsh

    du, dut, _, _ = ln("out_ln", R.dense_bwd_x(dpred, p["out.kernel"]), R.dense_bwd_x(dpredt, p["out.kernel"]), u[K],
                       ut[K], "out_ln.", None)
    grads[f"k{K - 1}.res.b.bias"] = R.dense_bwd_b(du)
    for k in range(K - 1, -1, -1):
        pre, fp = f"k{k}.res.", f"k{k}.film."
        acta, actta, actb, acttb = acts[k]
        e1pre, e1, e2, ss = film[k]
        grads[pre + "b.kernel"] = R.dense_bwd_w(actb, du) + R.dense_bwd_w(acttb, dut)
        dr1, dr1t, dsc_b, dsh_b = ln(f"ln_b[{k}]", R.dense_bwd_x(du, p[pre + "b.kernel"]),
                                     R.dense_bwd_x(dut, p[pre + "b.kernel"]), *r1s[k], pre + "ln_b.", ss)
        grads[pre + "a.bias"] = R.dense_bwd_b(dr1)
        grads[pre + "a.kernel"] = R.dense_bwd_w(acta, dr1) + R.dense_bwd_w(actta, dr1t)
        dxa, dxat, dsc_a, dsh_a = ln(f"ln_a[{k}]", R.dense_bwd_x(dr1, p[pre + "a.kernel"]),
                                     R.dense_bwd_x(dr1t, p[pre + "a.kernel"]), u[k], ut[k], pre + "ln_a.", ss,
                                     du[:, None])
        du, dut = dxa + du, dxat + dut
        grads[f"k{k - 1}.res.b.bias" if k > 0 else "in.bias"] = R.dense_bwd_b(du)
        dss = torch.cat([dsc_a + dsc_b, dsh_a + dsh_b], dim=-1)
        fg = R.film_generator_bwd(dss, enc, e1pre, e1, e2, p[fp + "ss.kernel"], p[fp + "d2.kernel"])
        for name in ("ss.kernel", "ss.bias", "d2.kernel", "d2.bias", "d1.kernel", "d1.bias"):
            grads[fp + name] = fg[name]
    grads["in.kernel"] = R.dense_bwd_w(xt, du) + R.dense_bwd_w(v, dut)
    return grads, launches


def _ncsn_inputs(B, C, seed):
    gen = torch.Generator().manual_seed(seed)
    x0 = torch.rand(B, C, generator=gen, dtype=F64) * 2 - 1
    eps = torch.randn(B, C, generator=gen, dtype=F64)
    v = torch.where(torch.rand(B, C, generator=gen, dtype=F64) < 0.5, 1.0, -1.0).to(F64)
    sig = torch.as_tensor(SIGMAS, dtype=F64)[torch.randint(0, len(SIGMAS), (B,), generator=gen)]
    return x0, sig, eps, v


def test_launch_rules_compose_to_the_reverse_over_reverse_gradient():
    C, Md, K, B = 8, 48, 2, 3
    p = SR.dense_ncsn_params(C, Md, K, seed=1)
    x0, sig, eps, v = _ncsn_inputs(B, C, 2)
    got, launches = ssm_step_fp64(p, x0, sig, eps, v, K, gb=B)
    assert [kind for kind, _, _ in launches] == ["out_ln", "ln_b[1]", "ln_a[1]", "ln_b[0]", "ln_a[0]"]
    leaves = {k: t.clone().requires_grad_(True) for k, t in p.items()}
    loss, _, _ = SR.ssm_loss_tensors(lambda a, s: O.dense_ncsn(leaves, a, s, num_layers=K, mlp_dims=Md), x0, sig, eps,
                                     v, "mean")
    loss.backward()
    assert sorted(got) == sorted(p)
    for name, leaf in leaves.items():
        err = _rel(got[name], leaf.grad)
        assert err < 1e-9, (name, err)


def test_gpu_rules_would_catch_a_dropped_term():
    """On the launches of the GPU base case's shape (C 64, mlp_dims 2048, two blocks, nine examples, sigmas drawn from
    the training schedule), a kernel that dropped any one term of the closed form would fail the GPU rule on the output
    the term feeds by more than ten times, on every launch that has the term.  dx is stored as bf16 after the residual
    adjoint is added (ln_a): its rule fails when the rel-L2 error, the share of elements beyond one bf16 spacing or the
    share not rounded to the nearest bf16 exceeds its bound; dscale is checked through the FiLM pair adjoint (B_DSS).
    The terms gr and gP move dx by only a few 1e-3 rel-L2, about the size of the bf16 rounding itself: the
    not-nearest share is the statistic that sees them."""
    from tests import test_gpu_backward_stages as BW
    from tests import test_gpu_ssm_backward_stages as G
    C, Md, K, B = 64, 2048, 2, 9
    p = SR.dense_ncsn_params(C, Md, K, seed=4)
    _, launches = ssm_step_fp64(p, *_ncsn_inputs(B, C, 7), K, gb=B)

    def bf16_rule(got, ref, far, not_nearest):
        """How many times over its bound the GPU bf16 rule would be for a device output `got` (before rounding)."""
        got = R.bf16_round(got)
        n = ref.numel()
        f_far = int(((got - ref).abs() > R.bf16_ulp(ref)).sum()) / n
        f_nn = int((got != R.bf16_round(ref)).sum()) / n
        return max(_rel(got, ref) / G.B_BF16, f_far / far, f_nn / not_nearest)

    worst = {}
    for kind, kw, dres in launches:
        full = closed_form(**kw)
        res = 0 if dres is None else dres
        far, nn = (BW.FAR_LN_B, BW.NOT_NEAREST_LN_B) if kind.startswith("ln_b") else (BW.FAR, BW.NOT_NEAREST)
        for term in TERMS:
            if kw["scale"] is None and term in ("swish2", "dscale_t"):
                continue   # out_ln: no FiLM, no activation
            cut = closed_form(**kw, drop=(term,))
            if term == "dscale_t":
                ratio = _rel(cut[4], full[4]) / G.B_DSS
            else:
                ratio = bf16_rule(cut[0] + res, full[0] + res, far, nn)
            print(f"{kind}: without {term} the GPU rule would be {ratio:.1f} x over its bound")
            worst[(kind, term)] = ratio
    low = {key: ratio for key, ratio in worst.items() if not ratio > 10}
    assert not low, low
