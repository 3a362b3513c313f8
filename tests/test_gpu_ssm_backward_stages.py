"""Every launch of the sliced score matching train step (DenseNCSN, csrc/backward.cu ssm_grads_impl) against a float64
restatement of THAT launch on the operands the device read.

The forward launches are those of test_gpu_forward_stages.check_forward with the tangent pass, plus q_sample, the
tangent cast and the loss.  The backward rules follow test_gpu_backward_stages.py: weight gradients are the primal
plus the tangent product; every dX GEMM runs on the primal and on the tangent adjoint; and each ssm_ln_bwd launch
(out_ln, then ln_b and ln_a of every block) is compared with backward_reference.ssm_ln_film_swish_bwd, the float64
autograd gradient of <g, out> + <g', out'> (pinned on the CPU by test_ssm_backward_reference.py).  The incoming g / g'
of a LayerNorm launch are the bf16-rounded float64 dX products of the device's adjoints; the fp32 residual adjoints
t.du32 / t.dut32, which the next ln_a overwrites, are carried in float64 from the top.  ln_a[0] reads t.g16 / t.gt16,
still in place after the call: they are checked as the outputs of the last two dX GEMMs and fed in exactly.  Each
case counts the launches of the call (Engine.launch_count) and asserts that the rules covered all of them, and that
every parameter tensor's gradient is covered by a rule.

The bounds are those of tests/test_gpu_backward_stages.py, plus one: B_DSS, the FiLM pair adjoint.  DenseNCSN has
one row per example, so each element of dss is the sum of two products of re-rounded incoming gradients, not a sum over
32 positions as in the DDPM file; its bound is about 3x the largest error measured.

Largest errors measured on an H100 80GB HBM3 (SXM, 700 W power limit) over all cases of this file / asserted bound:

- ssm_ln_bwd dx / dx' stored as bf16: rel-L2 1.86e-3 / B_BF16 2.5e-3; beyond one bf16 spacing 3.3e-4 / FAR 1.5e-3
  (ln_b 4.2e-3 / 1e-2); not the nearest bf16 2.4e-3 / NOT_NEAREST 8e-3 (ln_b 1.85e-2 / 4e-2)
- dgamma, dbeta and dbias sums fed by re-rounded dX products: at most 0.22 of b_wide_sums(rows) (7.6e-5 at 130 rows,
  2.4e-4 at 3 rows); ln_a[0], fed t.g16 / t.gt16 exactly: dgamma / dbeta 1.8e-7 / B_LN128 1e-5, dbias into in.bias
  6.1e-5 / B_LNWIDE 1e-4
- FiLM pair adjoint dss: 1.36e-4 / B_DSS 4e-4
- dX GEMM outputs t.g16 / t.gt16: rel-L2 1.73e-3 / 2.5e-3, not the nearest bf16 2.7e-3 / 8e-3
- weight gradients (primal + tangent product) 1.7e-7, FiLM generator 1.1e-5 / B_DW 2e-5
- seeds, loss, colsums 1.0e-7 / B_SEED 4e-7; dpred16 and dpredt16 bit-exact
"""
import numpy as np
import pytest
import torch

from oracle import ddpm_oracle as O
from tests import backward_reference as R
from tests import test_gpu_backward_stages as BW
from tests import test_gpu_forward_stages as FW

pytestmark = pytest.mark.gpu

F64 = torch.float64
B_EXACT, B_SEED, B_DW, B_BF16 = BW.B_EXACT, BW.B_SEED, BW.B_DW, BW.B_BF16
B_LN128, B_LNWIDE = BW.B_LN128, BW.B_LNWIDE
B_DSS = 4e-4   # FiLM pair adjoint of one row per example
SIGMAS = O.create_noise_schedule(1.0, 0.01, 15, "geometric")
_ceil = BW._ceil


def check_ssm_step(eng, rep, x0, sig, eps, vv, batch, gb):
    """The rules of one compute_ssm_grads call of `batch` examples with global batch gb on inputs (x0, sigma, eps, v)."""
    torch.cuda.synchronize()
    v = BW.PlanView(eng)
    cfg = eng.cfg
    C, Md, K, Bmax = cfg.channels, cfg.mlp_dims, cfg.num_layers, eng.max_batch
    M = batch
    assert C % 64 == 0   # the output projection is not padded
    s64, v64 = sig.to(F64), vv.to(F64)

    # ------------------------------------------------------------------ forward: draws, primal + tangent pass, loss
    xt = v.f32("xt", batch, C)
    rep.rel("q_sample -> xt", xt, x0.to(F64) + s64[:, None] * eps.to(F64), B_SEED)
    rep.exact("q_sample -> conditioning sigma", v.f32("tvec", batch), sig)
    rep.launch("q_sample")
    rep.exact("tangent cast -> xbt", v.b16("xbt", batch, C), R.bf16_round(v64))
    rep.launch("tangent_input")
    f = v.f32("eps_hat", batch, C)
    FW.check_forward(eng, rep, xt.float(), sig, batch, save=True, y=f, tangent=True)
    ft = v.f32("yt", batch, C)
    loss = 0.5 * (f * f).sum(1) + s64 * (v64 * ft).sum(1)
    rep.rel("ssm loss -> t.loss", v.f32("t.loss", batch), loss, B_SEED)
    rep.rel("ssm loss -> loss_sum, loss_sum / global batch", torch.cat([eng.loss_sum, eng.loss_mean]),
            torch.stack([loss.sum(), loss.sum() / gb]), B_SEED)
    # ------------------------------------------------------------------ the two seeds
    dpred32 = v.f32("t.dpred32", M, C)
    rep.rel("seed dpred32 = f / global batch", dpred32, f / gb, B_SEED)
    dz = v.b16("t.dpred16", M, C)
    rep.exact("seed dpred16 = bf16(dpred32)", dz, R.bf16_round(dpred32))
    dzt = v.b16("t.dpredt16", M, C)
    inv_gb = torch.tensor(1.0 / gb, dtype=torch.float32)   # fp32 products in the kernel's order
    rep.exact("seed dpredt16 = bf16(sigma v / global batch)", dzt,
              (sig[:, None] * vv * inv_gb.cuda()).bfloat16().to(F64))
    rep.launch("ssm_loss")

    # ------------------------------------------------------------------ output projection
    rep.grad(v, "out.bias", R.dense_bwd_b(dpred32), B_SEED, "colsum out.bias")
    rep.launch("colsum out.bias")

    def dw(rule, name, x, g, x_t, g_t):
        rep.grad(v, name, R.dense_bwd_w(x, g) + R.dense_bwd_w(x_t, g_t), B_DW, rule)
        rep.launch(rule + " primal")
        rep.launch(rule + " tangent")

    dw("dWout + tdWout", "out.kernel", v.b16("t.act_out", M, Md), dz, v.b16(f"t.actt{2 * K}", M, Md), dzt)
    stats_all = v.f32("stats", 2 * K + 1, _ceil(Bmax, 256), 2)[:, :M]
    ss_all = v.f32("ss", K, Bmax, 2 * Md)

    def dx_pair(rule, g, g_t, w):
        """The incoming adjoints of a LayerNorm launch: the dX GEMMs' float64 products, rounded to bf16 as stored."""
        rep.launch(rule + " primal")
        rep.launch(rule + " tangent")
        return R.bf16_round(R.dense_bwd_x(g, w)), R.bf16_round(R.dense_bwd_x(g_t, w))

    def ssm_ln(rule, g, gt, x, xt_, stats, pre, film_k, dres, dx16, dxt16, bias_name, b_sums, b_bias,
               far=BW.FAR, not_nearest=BW.NOT_NEAREST):
        """One ssm_ln_bwd launch.  Returns the float64 dx, dx' and the FiLM pair adjoint [dscale | dshift]."""
        gamma, beta = v.param(pre + "scale"), v.param(pre + "bias")
        sc = sh = None
        if film_k is not None:
            sc, sh = ss_all[film_k, :batch, :Md], ss_all[film_k, :batch, Md:]
        dx, dxt, dg, db, dsc, dsh = R.ssm_ln_film_swish_bwd(g[:, None], gt[:, None], x[:, None], xt_[:, None], gamma,
                                                            beta, sc, sh, stats[:, None],
                                                            None if film_k is None else "swish")
        dx, dxt = dx[:, 0], dxt[:, 0]
        if dres is not None:
            dx, dxt = dx + dres[0], dxt + dres[1]
        rep.bf16(f"{rule} dx -> {dx16}", v.b16(dx16, M, Md), dx, far=far, not_nearest=not_nearest)
        rep.bf16(f"{rule} dx' -> {dxt16}", v.b16(dxt16, M, Md), dxt, far=far, not_nearest=not_nearest)
        rep.grad(v, pre + "scale", dg, b_sums, f"{rule} dgamma")
        rep.grad(v, pre + "bias", db, b_sums, f"{rule} dbeta")
        rep.grad(v, bias_name, R.dense_bwd_b(dx), b_bias, f"{rule} dbias -> {bias_name}")
        rep.launch(rule)
        return dx, dxt, (None if film_k is None else torch.cat([dsc, dsh], dim=-1))

    # ------------------------------------------------------------------ final LayerNorm (no FiLM, no activation)
    w_out = v.b16("w.out_pad", Md, C)
    g, gt = dx_pair("dXout", dz, dzt, w_out)
    b_wide = BW.b_wide_sums(M)
    du, dut, _ = ssm_ln("out_ln", g, gt, v.f32(f"t.u{K}", M, Md), v.f32(f"t.ut{K}", M, Md), stats_all[2 * K],
                        "out_ln.", None, None, f"t.du16_{K}", f"t.dut16_{K}", f"k{K - 1}.res.b.bias", b_wide, b_wide)

    # ------------------------------------------------------------------ FiLM'd residual blocks
    for k in range(K - 1, -1, -1):
        pre = f"k{k}.res."
        du16, dut16 = v.b16(f"t.du16_{k + 1}", M, Md), v.b16(f"t.dut16_{k + 1}", M, Md)
        dw(f"dWb + tdWb[{k}]", pre + "b.kernel", v.b16(f"t.actb{k}", M, Md), du16, v.b16(f"t.actt{2 * k + 1}", M, Md),
           dut16)
        g, gt = dx_pair(f"dXb[{k}]", du16, dut16, v.w16(pre + "b.kernel"))
        _, _, dss_b = ssm_ln(f"ln_b[{k}]", g, gt, v.b16(f"t.r1_{k}", M, Md), v.f32(f"t.r1t{k}", M, Md),
                             stats_all[2 * k + 1], pre + "ln_b.", k, None, f"t.dr16t_{k}", f"t.drt16_{k}",
                             pre + "a.bias", b_wide, b_wide, far=BW.FAR_LN_B, not_nearest=BW.NOT_NEAREST_LN_B)
        dr16, drt16 = v.b16(f"t.dr16t_{k}", M, Md), v.b16(f"t.drt16_{k}", M, Md)
        dw(f"dWa + tdWa[{k}]", pre + "a.kernel", v.b16(f"t.acta{k}", M, Md), dr16, v.b16(f"t.actt{2 * k}", M, Md),
           drt16)
        wa = v.w16(pre + "a.kernel")
        g, gt = dx_pair(f"dXa[{k}]", dr16, drt16, wa)
        b_sums = b_bias = b_wide
        if k == 0:   # the last two dX outputs of the call are still in t.g16 / t.gt16: this launch's inputs are known
            g, gt = v.b16("t.g16", M, Md), v.b16("t.gt16", M, Md)
            rep.bf16("dXa[0] -> t.g16", g, R.dense_bwd_x(dr16, wa))
            rep.bf16("tdXa[0] -> t.gt16", gt, R.dense_bwd_x(drt16, wa))
            b_sums, b_bias = B_LN128, B_LNWIDE   # (dbias also sums the residual adjoint the test carries)
        du, dut, dss_a = ssm_ln(f"ln_a[{k}]", g, gt, v.f32(f"t.u{k}", M, Md), v.f32(f"t.ut{k}", M, Md),
                                stats_all[2 * k], pre + "ln_a.", k, (du, dut), f"t.du16_{k}", f"t.dut16_{k}",
                                f"k{k - 1}.res.b.bias" if k > 0 else "in.bias", b_sums, b_bias)
        dss = v.f32("t.dss", K, Bmax, 2 * Md)[k, :batch]
        rep.rel(f"FiLM pair adjoint dss[{k}] = ln_a + ln_b", dss, dss_a + dss_b, B_DSS)
        BW.film_generator_rules(v, rep, k, batch, dss)
        for name in ("colsum ss.bias", "cast dss16", "cast e2_16", "dWss", "dXss", "colsum d2.bias", "dW d2", "dX d2",
                     "colsum d1.bias", "dW d1"):
            rep.launch(f"film generator {name}[{k}]")

    # ------------------------------------------------------------------ input projection
    dw("dWin + tdWin", "in.kernel", v.b16("xb", M, C), v.b16("t.du16_0", M, Md), v.b16("xbt", M, C),
       v.b16("t.dut16_0", M, Md))
    fam = [(f"t.{n}{k}", Md) for n in ("du16_", "dut16_") for k in range(K + 1)]
    fam += [(f"t.{n}{k}", Md) for n in ("dr16t_", "drt16_") for k in range(K)]
    BW.reduction_tail_rules(v, rep, M, fam + [("t.dpred16", C), ("t.dpredt16", C)])
    return rep


# ----------------------------------------------------------------------------------------------------------------------
# cases
# ----------------------------------------------------------------------------------------------------------------------
def _engine(C, Md, K, batch, quiet=False, film_shift=None):
    from smd_b200 import Engine, ModelConfig
    eng = Engine(ModelConfig(arch="DenseNCSN", num_layers=K, channels=C, mlp_dims=Md), max_batch=batch, training=True)
    d = eng.flat_to_dict(eng.init_params(seed=4, perturb=0.05))
    if quiet:      # in.bias with a spread of 1e-2: the ln_a[0] row of an example with x~ = 0 has a variance of 1e-4
        b = d["in.bias"]
        d["in.bias"] = ((b - b.mean()) * (1e-2 / b.std())).astype(np.float32)
    if film_shift is not None:   # nearly every swish input of the tail in [-12, -3]
        rng = np.random.default_rng(3)
        for k in range(K):
            d[f"k{k}.film.ss.bias"][Md:] = rng.uniform(*film_shift, Md).astype(np.float32)
    eng.set_params(eng.dict_to_flat(d))
    eng.init_train_state()
    return eng


def _inputs(batch, C, seed, quiet=False):
    rng = np.random.default_rng(seed)
    x0 = rng.uniform(-1, 1, (batch, C)).astype(np.float32)
    eps = rng.standard_normal((batch, C)).astype(np.float32)
    vv = np.where(rng.random((batch, C)) < 0.5, 1.0, -1.0).astype(np.float32)
    sig = SIGMAS[rng.integers(0, 15, batch)].astype(np.float32)
    if quiet:
        x0[0] = 0.0
        eps[0] = 0.0
    return [torch.from_numpy(a).cuda() for a in (x0, sig, eps, vv)]


def check_ssm_call(eng, rep, inputs, batch, gb, launches):
    """Every rule of this file after a compute_ssm_grads call on `inputs` that counted `launches` kernel launches, then
    the launch count and the coverage of every parameter tensor."""
    check_ssm_step(eng, rep, *inputs, batch, gb)
    rep.expect_launches(launches)
    BW.assert_complete(eng, rep)
    rep.finish()


# The existing shape, DenseNCSN C 64 with two 2048-wide blocks at nine examples (the last 4-row CTA holds one row), is
# test_gpu_backward_stages.py's sliced score matching case, which runs check_ssm_call; the replay case reuses it.
BASE = (64, 2048, 2, 9)
CASES = {
    # name: (channels, mlp_dims, layers, batch, options)
    "vae": (512, 2048, 2, 130, dict(gb_mult=4)),        # reduction tail 130 -> 192; 33 CTAs of column atomics
    "narrow": (64, 256, 1, 5, {}),                      # 64-thread CTAs
    "cpt8_odd": (64, 2304, 1, 6, {}),                   # CPT = 8 with 288 threads (9 warps)
    "cpt8_max": (512, 4096, 2, 3, {}),                  # CPT = 8 with 512 threads; 1024-thread tangent forward
    "quiet": BASE + (dict(quiet=True),),                # example 0: ln_a[0] row variance ~1e-4, rstd ~100
    "film_shift": (64, 2048, 1, 9, dict(film_shift=(-10.0, -5.0))),
}


@pytest.mark.parametrize("case", list(CASES))
def test_every_ssm_backward_launch_matches_its_fp64_restatement(lib, case):
    C, Md, K, batch, opts = CASES[case]
    eng = _engine(C, Md, K, batch, quiet=opts.get("quiet", False), film_shift=opts.get("film_shift"))
    gb = opts.get("gb_mult", 1) * batch
    shares = (FW.FAR_SHIFT, FW.NOT_NEAREST_SHIFT) if "film_shift" in opts else (BW.FAR, BW.NOT_NEAREST)
    inputs = _inputs(batch, C, seed=7, quiet=opts.get("quiet", False))
    _, n = FW._counted(eng, lambda: eng.compute_ssm_grads(*inputs, global_batch=gb))
    if opts.get("quiet"):
        st = BW.PlanView(eng).f32("stats", 1, 2)[0] / Md
        var = float(st[1] - st[0] ** 2)
        print(f"[parity] quiet: ln_a[0] row 0 variance {var:.3e}")
        assert 5e-5 < var < 2e-4, var
    check_ssm_call(eng, FW.Report(case, shares), inputs, batch, gb, n)


def test_rules_hold_after_a_replayed_ssm_graph(lib):
    """On a capturable stream the first call runs eagerly, the second captures and the third replays the graph with new
    input tensors and a data-parallel global batch: the rules hold on the path training uses."""
    C, Md, K, batch = BASE
    eng = _engine(C, Md, K, batch)
    gb = 4 * batch
    stream = torch.cuda.Stream()
    for step in range(3):
        inputs = _inputs(batch, C, seed=50 + step)
        with torch.cuda.stream(stream):
            _, n = FW._counted(eng, lambda: eng.compute_ssm_grads(*inputs, global_batch=gb))
    check_ssm_call(eng, FW.Report("replay"), inputs, batch, gb, n)
