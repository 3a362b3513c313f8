"""Every launch of the backward pass against a float64 restatement of THAT launch on the operands the device read.

A training plan keeps almost every adjoint and every saved activation in a buffer of its own (smd_debug_buffer).
After one gradient call the rules below recompute, in float64 (tests/backward_reference.py), what each launch should
have written from the inputs it actually read, and compare with what it wrote.  Every rule restarts from device data,
so errors do not compound and the bounds are those of one launch: fp32 accumulation for the weight-gradient GEMMs and
column sums, one bfloat16 rounding for the stored adjoints.  The end-to-end gradient tests (test_gpu_train.py and
friends) check the composition at 2e-2; these rules say which launch is wrong, at 1e-4.

Quantities the plan overwrites before the call returns (the fp32 residual adjoints t.du32 / t.dh / t.dh2 and the bf16
dX output t.g16) are carried by the test in float64 from the top of the chain instead.

Each rule prints a "[parity]" line with the measured error next to the asserted bound (pytest -s).  The bounds are
about 3x the largest error measured on an H100 SXM (700 W limit) over the cases of this file.
"""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from oracle import ddpm_oracle as O
from smd_b200 import lib as L
from tests import backward_reference as R

pytestmark = pytest.mark.gpu

F64 = torch.float64

# rel-L2 bounds per class of output
B_EXACT = 0.0      # a copy or a cast: bit-identical
B_SEED = 4e-7      # elementwise fp32 arithmetic, column sums of persisted values, LayerNorm row statistics
B_DW = 2e-5        # bf16 operands, fp32 accumulation (also split-K with atomics), fp32 output; the fp32 SIMT products
B_LN128 = 1e-5     # parameter / bias sums of the 128-wide LayerNorm backward (its incoming gradient is fp32)
B_LNWIDE = 1e-4    # the same sums of a wide LayerNorm backward whose bf16 incoming gradient is known exactly
B_BF16 = 2.5e-3    # a value stored as bfloat16: the rounding alone measures 1.67e-3 on every such output
B_TF32 = 3e-3      # tf32 tensor-core products (attention backward at 32 positions) under the same bf16 store
B_TF32_SUM = 4e-4  # their column sums (qkv bias gradient)
FAR = 1.5e-3       # share of a bf16 output's elements allowed more than one bf16 spacing away from the reference
NOT_NEAREST = 8e-3  # share allowed to differ from the bf16 number nearest to the reference
FAR_LN_B, NOT_NEAREST_LN_B = 1e-2, 4e-2   # (ln_b: bf16 LayerNorm input and a re-rounded incoming gradient)


def b_wide_sums(rows):
    """Sums of a wide LayerNorm backward whose incoming gradient, the bf16 output of a 2048-long dX GEMM, is NOT kept:
    the reference rounds its own float64 product to bf16 and a fraction of a percent of the elements fall on the other
    side of a rounding boundary than the device's fp32 accumulation did.  That noise, not the kernel, sets the floor;
    it averages out over the rows summed (measured 4.3e-4 at 8 rows, 1.8e-4 at 130, 1.4e-5 at 4096)."""
    return max(4e-5, 4e-3 / math.sqrt(rows))


def _ceil(n, m):
    return (n + m - 1) // m * m


class _DeviceBytes:
    """A workspace region as a uint8 device array, for torch.as_tensor."""

    def __init__(self, ptr: int, nbytes: int):
        self.__cuda_array_interface__ = {"shape": (nbytes,), "typestr": "|u1", "data": (ptr, False), "strides": None,
                                         "version": 3}


class Report:
    """Collects the measured error of every rule of one case; finish() fails with all violated rules at once."""

    def __init__(self, case):
        self.case, self.failed, self.covered, self.rules = case, [], set(), 0

    def rel(self, rule, got, ref, bound, covers=None):
        got, ref = got.to(F64), ref.to(F64)
        assert got.shape == ref.shape, (rule, got.shape, ref.shape)
        err = float((got - ref).norm() / (ref.norm() + 1e-300))
        ok = err <= bound and math.isfinite(err) and float(ref.norm()) > 0.0
        print(f"[parity] {self.case} {rule}: rel_l2={err:.3e} bound={bound:.1e}{'' if ok else '  <-- FAILED'}")
        self.rules += 1
        if not ok:
            self.failed.append((rule, err, bound))
        if covers:
            self.covered.add(covers)

    def grad(self, eng_view, name, ref, bound, rule=None):
        self.rel(rule or f"grad {name}", eng_view.grad(name), ref, bound, covers=name)

    def bf16(self, rule, got, ref, bound=B_BF16, far=FAR, not_nearest=NOT_NEAREST):
        """A value stored as bfloat16: rel-L2; the share of elements more than one bf16 spacing from the reference; and
        the share that is not the bf16 number nearest to the reference (the statistic that notices a relative error of
        1e-4, far below the rounding)."""
        self.rel(rule, got, ref, bound)
        got = got.to(F64)
        n = ref.numel()
        f_far = int(((got - ref).abs() > R.bf16_ulp(ref)).sum()) / n
        f_nn = int((got != R.bf16_round(ref)).sum()) / n
        ok = f_far <= far and f_nn <= not_nearest
        print(f"[parity] {self.case} {rule}: beyond_1_bf16_ulp={f_far:.3e} allowed={far:.1e} "
              f"not_nearest_bf16={f_nn:.3e} allowed={not_nearest:.1e}{'' if ok else '  <-- FAILED'}")
        if not ok:
            self.failed.append((rule + " (bf16 elements off)", (f_far, f_nn), (far, not_nearest)))

    def zero(self, rule, t):
        nz = int((t != 0).sum())
        print(f"[parity] {self.case} {rule}: nonzero={nz}/{t.numel()}")
        self.rules += 1
        if nz:
            self.failed.append((rule, nz, 0))

    def finish(self):
        assert not self.failed, f"{self.case}: {len(self.failed)} of {self.rules} rules failed: {self.failed}"


class PlanView:
    """Typed float64 reads of the workspace regions, parameters, bf16 weight shadow and gradients of an engine."""

    def __init__(self, eng):
        self.eng = eng
        self.layout = {name: (off, shape) for name, off, shape in eng.layout}

    def raw(self, name, shape, dtype):
        ptr, nbytes = C.c_void_p(), C.c_size_t()
        L.check(self.eng.lib.smd_debug_buffer(self.eng._plan, name.encode(), C.byref(ptr), C.byref(nbytes)))
        need = int(np.prod(shape)) * torch.tensor([], dtype=dtype).element_size()
        assert need <= nbytes.value, (name, need, nbytes.value)
        raw = torch.as_tensor(_DeviceBytes(ptr.value, nbytes.value), device="cuda")
        return raw[:need].view(dtype).reshape(shape)

    def f32(self, name, *shape):
        return self.raw(name, shape, torch.float32).to(F64)

    def b16(self, name, *shape):
        return self.raw(name, shape, torch.bfloat16).to(F64)

    def _slice(self, flat, name):
        off, shape = self.layout[name]
        return flat[off:off + int(np.prod(shape))].reshape(shape).to(F64)

    def param(self, name):
        return self._slice(self.eng.params, name)

    def w16(self, name):
        """The bf16 copy of a weight the tensor-core GEMMs read (same offsets as the fp32 arena)."""
        return self._slice(self.raw("wshadow", (self.eng.arena_floats,), torch.bfloat16), name)

    def grad(self, name):
        return self._slice(self.eng.grads, name)


def check_stages(eng, batch, rep, eps=None, objective="ddpm", global_batch=None):
    """The stage rules after one gradient call of `batch` examples on `eng`.  objective: "ddpm" / "dsm" (eps given: the
    loss seed is checked) or "mdn" (TransformerMDN: every rule below the head adjoint).  Sliced score matching has a
    file of its own (test_gpu_ssm_backward_stages.py)."""
    torch.cuda.synchronize()
    v = PlanView(eng)
    cfg = eng.cfg
    dense = cfg.arch in ("DenseDDPM", "DenseNCSN")
    mdn = objective == "mdn"
    S, Cc, Md, H = eng.seq_len, cfg.channels, cfg.mlp_dims, cfg.num_heads
    Lt = 0 if dense else cfg.num_layers
    K = cfg.num_layers if dense else cfg.num_mlp_layers
    M, Bmax = batch * S, eng.max_batch
    gb = global_batch or batch
    if mdn:
        kc = cfg.mdn_components
        KCp, Kcp = _ceil(kc * Cc, 64), _ceil(kc, 64)
        Hp = 2 * KCp + Kcp
        heads = [("mdn.mu.", 0, kc * Cc), ("mdn.log_sigma.", KCp, kc * Cc), ("mdn.pi.", 2 * KCp, kc)]
    else:
        Hp = _ceil(Cc, 64)
        heads = [("out.", 0, Cc)]
    stats_all = v.f32("stats", 2 * K + 1, _ceil(Bmax * S, 256), 2)[:, :M]

    # ------------------------------------------------------------------ loss seed
    dz = v.b16("t.dpred16", M, Hp)
    if objective in ("ddpm", "dsm"):
        pred = v.f32("eps_hat", batch, S * Cc)
        e64 = eps.reshape(batch, S * Cc).to(F64)
        loss, dpred = (R.ddpm_loss_seed if objective == "ddpm" else R.dsm_loss_seed)(e64, pred, gb)
        dpred32 = v.f32("t.dpred32", M, Cc)
        rep.rel("loss seed dpred32", dpred32, dpred.reshape(M, Cc), B_SEED)
        rep.rel("loss seed dpred16 = bf16(dpred32)", dz[:, :Cc], R.bf16_round(dpred32), B_EXACT)
        rep.rel("loss seed per-example loss", v.f32("t.loss", batch), loss, B_SEED)
        rep.rel("loss seed loss_sum", eng.loss_sum.to(F64), loss.sum().reshape(1), B_SEED)
        rep.grad(v, "out.bias", R.dense_bwd_b(dpred32), B_SEED, "colsum out.bias")
    if not mdn and Hp > Cc:
        rep.zero("dpred16 pad columns", v.raw("t.dpred16", (M, Hp), torch.bfloat16)[:, Cc:])

    # ------------------------------------------------------------------ output projection / MDN head
    act_out = v.b16("t.act_out", M, Md)
    for pre, off, cols in heads:
        rep.grad(v, pre + "kernel", R.dense_bwd_w(act_out, dz[:, off:off + cols]), B_DW, f"dW {pre}kernel")
        if mdn:
            rep.grad(v, pre + "bias", R.dense_bwd_b(dz[:, off:off + cols]), B_SEED, f"colsum {pre}bias")

    def wide_ln(rule, g, x, stats, pre, film_k, dres, dx16_name, bias_name, b_sums, b_bias=None,
                far=FAR, not_nearest=NOT_NEAREST):
        """One launch of the wide LayerNorm (+ FiLM + swish) backward.  Returns the fp64 dx and (dscale, dshift)."""
        gamma, beta = v.param(pre + "scale"), v.param(pre + "bias")
        if film_k is None:
            dx, dg, db = R.layer_norm_bwd(g, x, gamma, stats)
            dss = None
        else:
            ss = v.f32("ss", K, Bmax, 2 * Md)[film_k, :batch]
            dx, dg, db, dsc, dsh = R.ln_film_swish_bwd(g.reshape(batch, S, Md), x.reshape(batch, S, Md), gamma, beta,
                                                       ss[:, :Md], ss[:, Md:], stats.reshape(batch, S, 2))
            dx, dss = dx.reshape(M, Md), torch.cat([dsc, dsh], dim=-1)
        if dres is not None:
            dx = dx + dres
        rep.bf16(f"{rule} dx -> {dx16_name}", v.b16(dx16_name, M, Md), dx, far=far, not_nearest=not_nearest)
        rep.grad(v, pre + "scale", dg, b_sums, f"{rule} dgamma")
        rep.grad(v, pre + "bias", db, b_sums, f"{rule} dbeta")
        rep.grad(v, bias_name, R.dense_bwd_b(dx), b_bias or b_sums, f"{rule} dbias -> {bias_name}")
        return dx, dss

    # ------------------------------------------------------------------ final LayerNorm
    for k in range(K + 1):
        rep.rel(f"stats of t.u{k}", stats_all[2 * k], R.row_stats(v.f32(f"t.u{k}", M, Md)), B_SEED)
    g = R.bf16_round(R.dense_bwd_x(dz, v.b16("w.out_pad", Md, Hp)))
    du, _ = wide_ln("out_ln", g, v.f32(f"t.u{K}", M, Md), stats_all[2 * K], "out_ln.", None, None, f"t.du16_{K}",
                    f"k{K - 1}.res.b.bias", B_LNWIDE)   # (a short reduction: the re-rounded dX output agrees)

    # ------------------------------------------------------------------ FiLM'd residual blocks
    for k in range(K - 1, -1, -1):
        pre = f"k{k}.res."
        du16_next, dr16t = v.b16(f"t.du16_{k + 1}", M, Md), v.b16(f"t.dr16t_{k}", M, Md)
        rep.grad(v, pre + "b.kernel", R.dense_bwd_w(v.b16(f"t.actb{k}", M, Md), du16_next), B_DW, f"dWb[{k}]")
        rep.grad(v, pre + "a.kernel", R.dense_bwd_w(v.b16(f"t.acta{k}", M, Md), dr16t), B_DW, f"dWa[{k}]")
        # TransformerMDN has no FiLM generator: its blocks read the identity pair kept in block 0
        film_k = 0 if mdn else k
        g = R.bf16_round(R.dense_bwd_x(du16_next, v.w16(pre + "b.kernel")))
        _, dss_b = wide_ln(f"ln_b[{k}]", g, v.b16(f"t.r1_{k}", M, Md), stats_all[2 * k + 1], pre + "ln_b.", film_k,
                           None, f"t.dr16t_{k}", pre + "a.bias", b_wide_sums(M), far=FAR_LN_B,
                           not_nearest=NOT_NEAREST_LN_B)
        g = R.bf16_round(R.dense_bwd_x(dr16t, v.w16(pre + "a.kernel")))
        b_sums = b_bias = b_wide_sums(M)
        if k == 0:   # the last dX output of the call is still in t.g16: this launch's incoming gradient is known
            g16 = v.b16("t.g16", M, Md)
            rep.bf16("dXa[0] -> t.g16", g16, R.dense_bwd_x(dr16t, v.w16(pre + "a.kernel")))
            g, b_sums, b_bias = g16, B_LN128, B_LNWIDE   # (dbias also sums the residual adjoint the test carries)
        prev_bias = f"k{k - 1}.res.b.bias" if k > 0 else ("post.bias" if Lt else "in.bias")
        du, dss_a = wide_ln(f"ln_a[{k}]", g, v.f32(f"t.u{k}", M, Md), stats_all[2 * k], pre + "ln_a.", film_k, du,
                            f"t.du16_{k}", prev_bias, b_sums, b_bias)
        if mdn:
            continue
        dss = v.f32("t.dss", K, Bmax, 2 * Md)[k, :batch]
        rep.rel(f"FiLM pair adjoint dss[{k}]", dss, dss_a + dss_b, b_wide_sums(S) / 4)
        film_generator_rules(v, rep, k, batch, dss)

    du16_0 = v.b16("t.du16_0", M, Md)
    if dense:
        # ---------------------------------------------------------- input projection of the dense models
        Cp = _ceil(Cc, 64)
        rep.grad(v, "in.kernel", R.dense_bwd_w(v.b16("xb", M, Cp)[:, :Cc], du16_0), B_DW, "dWin")
    else:
        # ---------------------------------------------------------- post dense + post LayerNorm
        def ln128(rule, g, h_name, pre, dres, dx16_name, bias_name):
            dx, dg, db = R.layer_norm_bwd(g, v.f32(h_name, M, 128), v.param(pre + "scale"))
            if dres is not None:
                dx = dx + dres
            if dx16_name:
                rep.bf16(f"{rule} dx -> {dx16_name}", v.b16(dx16_name, M, 128), dx)
            rep.grad(v, pre + "scale", dg, B_LN128, f"{rule} dgamma")
            rep.grad(v, pre + "bias", db, B_LN128, f"{rule} dbeta")
            rep.grad(v, bias_name, R.dense_bwd_b(dx), B_LN128, f"{rule} dbias -> {bias_name}")
            return dx

        rep.grad(v, "post.kernel", R.dense_bwd_w(v.b16("t.a_post", M, 128), du16_0), B_DW, "dWpost")
        dh = ln128("post_ln", R.dense_bwd_x(du16_0, v.w16("post.kernel")), f"t.h{2 * Lt}", "post_ln.", None,
                   f"t.dh16a{Lt - 1}", f"l{Lt - 1}.ffn2.bias")
        for l in range(Lt - 1, -1, -1):
            pre = f"l{l}."
            dh16a = v.b16(f"t.dh16a{l}", M, 128)
            # FFN
            ref = R.dense_bwd_x(dh16a, v.w16(pre + "ffn2.kernel")) * R.gelu_tanh_grad(v.b16(f"t.hpre{l}", M, Md))
            dr16 = v.b16(f"t.dr16_{l}", M, Md)
            rep.bf16(f"dX2[{l}] x gelu'(hpre) -> t.dr16_{l}", dr16, ref)
            rep.grad(v, pre + "ffn2.kernel", R.dense_bwd_w(v.b16(f"t.hid{l}", M, Md), dh16a), B_DW, f"dW2[{l}]")
            rep.grad(v, pre + "ffn1.bias", R.dense_bwd_b(dr16), B_SEED, f"colsum ffn1.bias[{l}]")
            rep.grad(v, pre + "ffn1.kernel", R.dense_bwd_w(v.b16(f"t.a2_{l}", M, 128), dr16), B_DW, f"dW1[{l}]")
            dh = ln128(f"ln2[{l}]", R.dense_bwd_x(dr16, v.w16(pre + "ffn1.kernel")), f"t.h{2 * l + 1}", pre + "ln2.",
                       dh, f"t.dh16b{l}", pre + "attn.out.bias")
            # attention
            dh16b = v.b16(f"t.dh16b{l}", M, 128)
            rep.grad(v, pre + "attn.out.kernel", R.dense_bwd_w(v.b16(f"t.o{l}", M, 128), dh16b), B_DW, f"dWo[{l}]")
            probs = v.f32(f"t.probs{l}", batch, H, S, S)
            if mdn:
                rep.zero(f"probs[{l}] above the diagonal", probs * torch.ones_like(probs[0, 0]).triu(1))
            d_o = R.dense_bwd_x(dh16b, v.w16(pre + "attn.out.kernel"))
            dqkv = R.attention_bwd(v.f32(f"t.qkv{l}", batch, S, 384), probs, d_o.reshape(batch, S, 128), H)
            dqkv = dqkv.reshape(M, 384)
            tf32 = S == 32 and (128 // H) % 8 == 0
            dqkv16 = v.b16(f"t.dqkv16_{l}", M, 384)
            if tf32:
                rep.rel(f"attention bwd[{l}] (tf32) -> t.dqkv16_{l}", dqkv16, dqkv, B_TF32)
            else:
                rep.bf16(f"attention bwd[{l}] -> t.dqkv16_{l}", dqkv16, dqkv)
            rep.grad(v, pre + "attn.qkv.bias", R.dense_bwd_b(dqkv), B_TF32_SUM if tf32 else B_SEED,
                     f"attention bwd[{l}] dbias")
            rep.grad(v, pre + "attn.qkv.kernel", R.dense_bwd_w(v.b16(f"t.a1_{l}", M, 128), dqkv16), B_DW, f"dWqkv[{l}]")
            dh = ln128(f"ln1[{l}]", R.dense_bwd_x(dqkv16, v.w16(pre + "attn.qkv.kernel")), f"t.h{2 * l}", pre + "ln1.",
                       dh, f"t.dh16a{l - 1}" if l > 0 else None, f"l{l - 1}.ffn2.bias" if l > 0 else "in.bias")
        dh_dev = v.f32("t.dh", M, 128)
        rep.rel("trunk residual adjoint -> t.dh", dh_dev, dh, B_LN128)
        # ---------------------------------------------------------- embedding
        rep.grad(v, "in.kernel", R.dense_bwd_w(v.f32("xt", M, Cc), dh_dev), B_SEED * 2, "embedding bwd")

    # ------------------------------------------------------------------ reduction-tail rows of the MN-major operands
    fam = [(f"t.du16_{k}", Md) for k in range(K + 1)] + [(f"t.dr16t_{k}", Md) for k in range(K)]
    fam += [("t.dpred16", Hp)]
    for l in range(Lt):
        fam += [(f"t.dh16a{l}", 128), (f"t.dh16b{l}", 128), (f"t.dr16_{l}", Md), (f"t.dqkv16_{l}", 384)]
    reduction_tail_rules(v, rep, M, fam)
    return rep


def film_generator_rules(v, rep, k, batch, dss):
    """The FiLM generator backward of block k (ten launches on the side stream) from the device's pair adjoint dss."""
    Md = v.eng.cfg.mlp_dims
    Bk = _ceil(batch, 64)
    fp = f"k{k}.film."
    dss16, e2_16 = R.bf16_round(dss), R.bf16_round(v.f32(f"t.e2_{k}", batch, 512))
    f = R.film_generator_bwd(dss16, v.f32("enc", batch, 128), v.f32(f"t.e1pre{k}", batch, 512),
                             v.f32(f"t.e1_{k}", batch, 512), e2_16, v.w16(fp + "ss.kernel"),
                             v.param(fp + "d2.kernel"))
    rep.grad(v, fp + "ss.bias", R.dense_bwd_b(dss), B_SEED, f"colsum film.ss.bias[{k}]")
    rep.grad(v, fp + "ss.kernel", f["ss.kernel"], B_DW, f"dWss[{k}]")
    for name in ("d2.bias", "d2.kernel", "d1.bias", "d1.kernel"):
        rep.grad(v, fp + name, f[name], B_DW, f"film generator {name}[{k}]")
    if k == 0:   # the generator's scratch buffers hold the block that ran last
        rep.rel("film generator dss16 = bf16(dss)", v.b16("t.dss16", batch, 2 * Md), dss16, B_EXACT)
        rep.rel("film generator e2_16 = bf16(e2)", v.b16("t.e2_16", batch, 512), e2_16, B_EXACT)
        rep.rel("film generator dXss -> t.de2", v.f32("t.de2", batch, 512), f["de2"], B_DW)
        rep.rel("film generator dX d2 -> t.de", v.f32("t.de", batch, 512), f["de1"], B_DW)
        if Bk != batch:
            rep.zero("tail rows of t.dss16", v.raw("t.dss16", (Bk, 2 * Md), torch.bfloat16)[batch:])
            rep.zero("tail rows of t.e2_16", v.raw("t.e2_16", (Bk, 512), torch.bfloat16)[batch:])


def reduction_tail_rules(v, rep, M, fam):
    """Rows [M, Mk) of the MN-major gradient operands fam = [(name, columns)] are zero (bwd_begin)."""
    Mk = _ceil(M, 64)
    if Mk == M:
        return
    bad = [n for n, cols in fam if bool((v.raw(n, (Mk, cols), torch.bfloat16)[M:] != 0).any())]
    print(f"[parity] {rep.case} rows [{M}, {Mk}) of {len(fam)} gradient operands: nonzero in {bad}")
    rep.rules += 1
    if bad:
        rep.failed.append(("reduction-tail rows not zero", bad, []))


def assert_complete(eng, rep):
    """Every tensor of the parameter arena got its gradient checked by some rule."""
    names = [name for name, _, _ in eng.layout]
    assert len(names) == eng.lib.smd_num_tensors(eng._plan)
    missing = [n for n in names if n not in rep.covered]
    print(f"[parity] {rep.case} parameter tensors: {len(names)}, not covered by a rule: {missing}")
    assert not missing, missing


# ----------------------------------------------------------------------------------------------------------------------
# cases
# ----------------------------------------------------------------------------------------------------------------------
def _draws(batch, shape, seed):
    rng = np.random.default_rng(seed)
    x0 = rng.uniform(-1, 1, (batch, *shape)).astype(np.float32)
    used = rng.uniform(0.05, 0.99, (batch,)).astype(np.float32)
    eps = rng.standard_normal((batch, *shape)).astype(np.float32)
    return [torch.from_numpy(a).cuda() for a in (x0, used, eps)]


def _engine(arch, kw, max_batch, seed=2):
    from smd_b200 import Engine, ModelConfig
    eng = Engine(ModelConfig(arch=arch, **kw), max_batch=max_batch, training=True)
    eng.set_params(eng.init_params(seed=seed, perturb=0.05))
    eng.init_train_state()
    return eng


def _shape(arch, kw):
    return (kw.get("seq_len", 32), kw["channels"]) if arch.startswith("Transformer") else (kw["channels"],)


CASES = {
    # name: (arch, ModelConfig kwargs, batch)
    "L2_H8_K2_C42_b6": ("TransformerDDPM", dict(num_layers=2, num_heads=8, num_mlp_layers=2, channels=42), 6),
    # 96 tokens: reduction length 128 with 32 zeroed tail rows, output projection padded to 192 columns
    "L2_H16_K3_C146_b3": ("TransformerDDPM", dict(num_layers=2, num_heads=16, num_mlp_layers=3, channels=146), 3),
    "H4_b3": ("TransformerDDPM", dict(num_layers=1, num_heads=4, num_mlp_layers=1, channels=42), 3),
    "H32_b3": ("TransformerDDPM", dict(num_layers=1, num_heads=32, num_mlp_layers=1, channels=42), 3),   # SIMT attention
    "H8_b1": ("TransformerDDPM", dict(num_layers=1, num_heads=8, num_mlp_layers=1, channels=42), 1),
    "S64_H8_b3": ("TransformerDDPM", dict(num_layers=1, num_heads=8, num_mlp_layers=1, channels=42, seq_len=64), 3),
    "S128_H16_b2": ("TransformerDDPM", dict(num_layers=1, num_heads=16, num_mlp_layers=1, channels=42, seq_len=128), 2),
    "dense_C512_b8": ("DenseDDPM", dict(num_layers=2, channels=512), 8),
    "dense_C512_b130": ("DenseDDPM", dict(num_layers=2, channels=512), 130),   # 130 rows: reduction length 192
}


@pytest.mark.parametrize("case", list(CASES))
def test_every_backward_launch_matches_its_fp64_restatement(lib, case):
    arch, kw, batch = CASES[case]
    eng = _engine(arch, kw, batch)
    x0, used, eps = _draws(batch, _shape(arch, kw), seed=21)
    eng.compute_grads(x0, used, eps)
    rep = check_stages(eng, batch, Report(case), eps=eps)
    assert_complete(eng, rep)
    rep.finish()


BASE_B128 = ("TransformerDDPM", dict(num_layers=6, num_heads=8, num_mlp_layers=2, channels=42), 128)

# Runs in a process of its own: a profiler session leaves CUPTI attached to the process, and a later session in the same
# process (tests/test_gpu_gemm_wide.py) then came back without kernel events.
_PROFILE_BACKWARD = """
import sys, torch
from torch.profiler import ProfilerActivity, profile
from tests import test_gpu_backward_stages as T
arch, kw, batch = T.BASE_B128
eng = T._engine(arch, kw, batch)
inputs = T._draws(batch, T._shape(arch, kw), seed=22)
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    eng.compute_grads(*inputs)
    torch.cuda.synchronize()
for e in prof.events():
    if "gemm_bf16_wgmma" in e.name:
        print("KERNEL", e.name)
"""


def test_benchmarked_shape_runs_the_wide_tiles_and_the_largest_split_counts(lib):
    """base L6/H8/K2/C42 at batch 128 (4096 tokens): the res-block dW and dX GEMMs take the 128 x 256 layout and the
    trunk's dW GEMMs their largest split-K counts."""
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    flags = ["-s"] if sys.flags.no_user_site else []
    r = subprocess.run([sys.executable, *flags, "-c", _PROFILE_BACKWARD], cwd=root, capture_output=True, text=True,
                       timeout=200)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    kernels = [ln.split(" ", 1)[1] for ln in r.stdout.splitlines() if ln.startswith("KERNEL ")]
    wide = sum("gemm_bf16_wgmma_wide_kernel" in n for n in kernels)
    print(f"[parity] base_b128 wgmma GEMM launches: {len(kernels)}, of them 128x256: {wide}")
    assert wide >= 8, kernels            # dWb, dXb, dWa, dXa of both res-blocks at least
    arch, kw, batch = BASE_B128
    eng = _engine(arch, kw, batch)
    x0, used, eps = _draws(batch, _shape(arch, kw), seed=22)
    eng.compute_grads(x0, used, eps)
    rep = check_stages(eng, batch, Report("base_b128"), eps=eps)
    assert_complete(eng, rep)
    rep.finish()


def test_small_batch_after_a_larger_one_on_the_same_plan(lib):
    """Rows [M, Mk) of every gradient operand still hold the previous, larger step's adjoints unless bwd_begin zeroes
    them: after each step of 6, 3, 5, 1 examples on one plan the stage rules hold and the gradients are those of a fresh
    engine given only that step (up to the order of the split-K atomics)."""
    from tests.util import rel_l2
    arch, kw = "TransformerDDPM", dict(num_layers=2, num_heads=8, num_mlp_layers=2, channels=42)
    eng = _engine(arch, kw, 6)
    for step, batch in enumerate((6, 3, 5, 1)):
        x0, used, eps = _draws(batch, _shape(arch, kw), seed=30 + step)
        eng.compute_grads(x0, used, eps)
        rep = check_stages(eng, batch, Report(f"sequence step{step} b{batch}"), eps=eps)
        assert_complete(eng, rep)
        fresh = _engine(arch, kw, 6)
        fresh.compute_grads(x0, used, eps)
        torch.cuda.synchronize()
        err = rel_l2(eng.grads, fresh.grads)
        print(f"[parity] sequence step{step} b{batch} gradients vs a fresh engine: rel_l2={err:.3e} bound=1.0e-05")
        assert err < 1e-5, (step, batch, err)
        rep.finish()
        del fresh


def test_dense_small_batch_after_a_larger_one(lib):
    """The same for the dense model, whose FiLM generator GEMMs reduce over the batch rounded up to 64."""
    from tests.util import rel_l2
    arch, kw = "DenseDDPM", dict(num_layers=2, channels=512)
    eng = _engine(arch, kw, 130)
    for step, batch in enumerate((130, 70, 3)):
        x0, used, eps = _draws(batch, _shape(arch, kw), seed=40 + step)
        eng.compute_grads(x0, used, eps)
        rep = check_stages(eng, batch, Report(f"dense sequence step{step} b{batch}"), eps=eps)
        fresh = _engine(arch, kw, 130)
        fresh.compute_grads(x0, used, eps)
        torch.cuda.synchronize()
        err = rel_l2(eng.grads, fresh.grads)
        print(f"[parity] dense sequence step{step} b{batch} gradients vs a fresh engine: rel_l2={err:.3e} bound=1.0e-05")
        assert err < 1e-5, (step, batch, err)
        rep.finish()
        del fresh


def test_rules_hold_after_a_replayed_cuda_graph(lib):
    """On a capturable stream the first call runs eagerly, the second captures and the third replays the graph: the
    buffers are checked on the path training uses, with new input tensors every step and a data-parallel global batch."""
    arch, kw, batch = CASES["L2_H8_K2_C42_b6"]
    eng = _engine(arch, kw, batch)
    stream = torch.cuda.Stream()
    for step in range(3):
        x0, used, eps = _draws(batch, _shape(arch, kw), seed=50 + step)
        with torch.cuda.stream(stream):
            eng.compute_grads(x0, used, eps, global_batch=4 * batch)
        torch.cuda.synchronize()
    rep = check_stages(eng, batch, Report("graph replay"), eps=eps, global_batch=4 * batch)
    assert_complete(eng, rep)
    rep.finish()


def _ncsn(batch, channels=64):
    eng = _engine("DenseNCSN", dict(num_layers=2, channels=channels), batch, seed=4)
    rng = np.random.default_rng(7)
    sigmas = O.create_noise_schedule(1.0, 0.01, 15, "geometric")
    x0 = rng.uniform(-1, 1, (batch, channels)).astype(np.float32)
    eps = rng.standard_normal((batch, channels)).astype(np.float32)
    vv = np.where(rng.random((batch, channels)) < 0.5, 1.0, -1.0).astype(np.float32)
    sig = sigmas[rng.integers(0, 15, batch)].astype(np.float32)
    return eng, [torch.from_numpy(a).cuda() for a in (x0, sig, eps, vv)]


def test_denoising_score_matching_seed_and_output_projection(lib):
    """DenseNCSN with the DSM objective: the seed is (raw + eps) / global batch on the raw network output, and every
    rule below it is that of the dense model."""
    batch = 9
    eng, (x0, sig, eps, _) = _ncsn(batch)
    eng.compute_dsm_grads(x0, sig, eps)
    rep = check_stages(eng, batch, Report("dsm"), eps=eps, objective="dsm")
    assert_complete(eng, rep)
    rep.finish()


def test_sliced_score_matching_weight_gradients_sum_primal_and_tangent_products(lib):
    """SSM accumulates the tangent product onto the primal product in place (the GEMM's residual is its own output).
    DenseNCSN C 64, two blocks, nine examples: every rule of test_gpu_ssm_backward_stages.py (which holds the other
    SSM shapes), the second-order LayerNorm backward included, and no parameter tensor left out."""
    from tests import test_gpu_forward_stages as FW
    from tests import test_gpu_ssm_backward_stages as SSM
    batch = 9
    eng, inputs = _ncsn(batch)
    _, n = FW._counted(eng, lambda: eng.compute_ssm_grads(*inputs))
    SSM.check_ssm_call(eng, FW.Report("ssm"), inputs, batch, batch, n)


def test_transformer_mdn_trunk_and_head(lib):
    """TransformerMDN: the three head weight gradients are column slices of one adjoint dZ, the blocks run without a
    FiLM generator, and the causal attention backward reads probabilities that are exactly zero above the diagonal."""
    from smd_b200 import Engine, ModelConfig
    kw = dict(num_layers=2, num_heads=8, num_mlp_layers=2, channels=42, mdn_components=10)
    batch = 3
    eng = Engine(ModelConfig(arch="TransformerMDN", **kw), max_batch=batch, training=True)
    eng.set_params(eng.init_params(seed=2, perturb=0.05))
    eng.init_train_state()
    x = torch.from_numpy(np.random.default_rng(8).uniform(-1, 1, (batch, 32, 42)).astype(np.float32)).cuda()
    eng.compute_mdn_grads(x)
    rep = check_stages(eng, batch, Report("mdn"), objective="mdn")
    assert_complete(eng, rep)
    rep.finish()
