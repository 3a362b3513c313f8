"""Every launch of the forward pass against a float64 restatement of THAT launch on the operands the device read.

On a training plan every index of a forward-activation family has a workspace region of its own (smd_debug_buffer),
and an inference call (smd_forward) on such a plan still takes the inference path -- the fused attention block, the
fused FFN, no saved probabilities -- bit for bit as an inference plan (test_gpu_plan_buffers.py).  So after one
forward call the rules below read the input and the output of every launch, recompute the output in float64
(tests/forward_reference.py) from the inputs the device actually read, and compare.  Every rule restarts from device
data, so errors do not compound and a rule names the launch that is wrong.  Each case also counts the kernel launches
of the call (Engine.launch_count) and asserts that the rules covered exactly that many: a launch added to the forward
pass without a rule fails here.

Bounds are those of tests/test_gpu_backward_stages.py where they apply (fp32 accumulation B_DW, fp32 elementwise and
row statistics B_SEED, one bf16 rounding B_BF16 with its far / not-nearest shares, tf32 attention B_TF32).  New ones:

- B_ATTN_BLOCK, B_FFN_FUSED: the fused attention block and the fused FFN keep o / the hidden activation on chip as bf16
  operands.  The restatement rounds its own float64 o / hidden to bf16; a fraction of the elements round the other way
  than the device's fp32 value did, which sets the floor.
- C_ACT: swish (ln_film_act) and tanh-GELU (FFN-up epilogue, fused FFN) use tanh.approx.f32, whose relative error the
  PTX ISA gives as about 2^-11.  Both are h + h tanh(.) with h = v / 2, so every activation stored as bf16 must satisfy
  |got - ref| <= ulp_bf16(ref) / 2 + PRE_SLACK rms(v) + C_ACT |v|, with v the pre-activation recomputed in float64 and
  PRE_SLACK rms(v) an allowance for the fp32 rounding of v itself; C_ACT = 2^-12 is the documented bound.  The
  far / not-nearest shares of these outputs are those of any bf16 output (FAR, NOT_NEAREST), except in one case whose
  FiLM shift puts nearly every swish input in [-12, -3].  There 0.5 + 0.5 tanh is a difference of nearly equal
  numbers, and swishf is NOT faithful to bf16: about 10 % of its outputs are more than one bf16 spacing from the exact
  swish and a quarter are not the nearest bf16 number (FAR_SHIFT, NOT_NEAREST_SHIFT).  The absolute error stays inside
  the c |v| contract above, which is what the consumers (the res-block GEMMs, where these inputs contribute outputs of
  about 1e-3) can see.
- Quiet rows: one case gives position 0 of every sample a trunk row variance of about 1e-4, where LayerNorm's eps
  (1e-6) matters at the 1 % level; its LayerNorm outputs are held to the same bf16 rules.

Largest errors measured on an H100 80GB HBM3 (SXM, 700 W power limit) over all cases of this file / asserted bound:

- fp32 outputs of bf16-operand GEMMs, FiLM generator and table, embed, stats partials: 7.5e-6 / B_DW 2e-5
- LayerNorm statistics totals, noise encoding, reverse step, SSM loss: 1.4e-7 / B_SEED 4e-7
- bf16 outputs (LayerNorm epilogues, res-a, tangent pass): 1.69e-3 / B_BF16 2.5e-3; elements beyond one spacing
  2.9e-4 / FAR 1.5e-3; not the nearest bf16 2.5e-3 / NOT_NEAREST 8e-3
- tf32 attention output 1.71e-3 / B_TF32 3e-3; its probabilities 3.3e-4 / 3e-3; SIMT probabilities 1.1e-7 / 4e-7
- fused attention block 1.71e-5 / B_ATTN_BLOCK 5e-5; fused FFN 4.69e-5 / B_FFN_FUSED 1.5e-4
- activations: rel-L2 1.71e-3 / 2.5e-3; max (|err| - ulp/2 - slack) / |v| 2.5e-8 / C_ACT 2.4e-4 (the c |v| term is
  never needed: every error fits inside half a spacing plus the pre-activation slack); shares beyond one spacing
  2.0e-4 / 1.5e-3, not the nearest 1.6e-3 / 8e-3; in the shifted case with inputs in [-12, -3] 9.5e-2 / 0.3 beyond one
  spacing and 0.25 / 0.75 not the nearest
"""
import ctypes as C
import time

import numpy as np
import pytest
import torch

from oracle import ddpm_oracle as O
from smd_b200 import lib as L
from tests import forward_reference as F
from tests import test_gpu_backward_stages as BW

pytestmark = pytest.mark.gpu

F64 = torch.float64
B_EXACT, B_SEED, B_DW, B_BF16, B_TF32 = BW.B_EXACT, BW.B_SEED, BW.B_DW, BW.B_BF16, BW.B_TF32
B_ATTN_BLOCK = 5e-5     # fused attention block: fp32 attention, o rounded to bf16 on chip
B_FFN_FUSED = 1.5e-4    # fused FFN: GELU through tanh.approx, hidden rounded to bf16 on chip
C_ACT = 2.0 ** -12      # tanh.approx.f32: relative error 2^-11 -> |v| 2^-12 on swish / GELU
PRE_SLACK = 2.0 ** -16  # fp32 error of the pre-activation itself, relative to its rms (absolute, per element)
FAR_SHIFT, NOT_NEAREST_SHIFT = 0.3, 0.75   # activation shares when nearly every swish input is in [-12, -3]

_ceil = BW._ceil


class Report(BW.Report):
    """The backward file's Report, plus the launches the rules cover and the activation contract."""

    def __init__(self, case, act_shares=(BW.FAR, BW.NOT_NEAREST)):
        super().__init__(case)
        self.launches = []
        self.act_shares = act_shares

    def launch(self, name):
        self.launches.append(name)

    def act(self, rule, got, ref, pre, c=C_ACT):
        """A bf16 output of swish / GELU: the bf16 rule with the activation shares, and the per-element bound."""
        self.bf16(rule, got, ref, far=self.act_shares[0], not_nearest=self.act_shares[1])
        slack = PRE_SLACK * float(pre.pow(2).mean().sqrt())
        ex = float(F.activation_excess(got.to(F64), ref, pre, slack).max())
        ok = ex <= c
        print(f"[parity] {self.case} {rule}: max (|err| - ulp/2 - slack) / |v| = {ex:.3e} bound={c:.2e}"
              f"{'' if ok else '  <-- FAILED'}")
        self.rules += 1
        if not ok:
            self.failed.append((rule + " (activation bound)", ex, c))

    def exact(self, rule, got, ref):
        ok = bool(torch.equal(got.to(F64), ref.to(F64)))
        n = int((got.to(F64) != ref.to(F64)).sum())
        print(f"[parity] {self.case} {rule}: differing={n}/{ref.numel()}{'' if ok else '  <-- FAILED'}")
        self.rules += 1
        if not ok:
            self.failed.append((rule, n, 0))

    def expect_launches(self, counted):
        n = len(self.launches)
        ok = n == counted
        print(f"[parity] {self.case} launches: counted={counted} covered by rules={n}{'' if ok else '  <-- FAILED'}")
        if not ok:
            self.failed.append(("launch count", counted, self.launches))


def check_forward(eng, rep, x, t, batch, *, save, bcast=False, y=None, table_row=None, tangent=False):
    """The rules of one forward call of `batch` examples on input x (device), conditioning t (device; one value when
    bcast) and raw network output y (device).  save: the call was a training-save forward.  table_row: the FiLM rows
    came from the sampler's table (no generator launches).  tangent: the DenseNCSN tangent pass ran alongside."""
    torch.cuda.synchronize()
    v = BW.PlanView(eng)
    cfg = eng.cfg
    dense = cfg.arch in ("DenseDDPM", "DenseNCSN")
    mdn = cfg.arch == "TransformerMDN"
    S, Cc, Md, H = eng.seq_len, cfg.channels, cfg.mlp_dims, cfg.num_heads
    Lt = 0 if dense else cfg.num_layers
    K = cfg.num_layers if dense else cfg.num_mlp_layers
    M, Bmax = batch * S, eng.max_batch
    Mp = _ceil(Bmax * S, 256)
    P, W = v.param, v.w16
    stats_all = v.f32("stats", 2 * K + 1, Mp, 2)[:, :M]
    xin = x.reshape(M, Cc).to(F64)
    # tables the plan builds once: checked against the oracle's, so that a launch reading them cannot agree with itself
    rep.rel("frequency table freqs", v.f32("freqs", 64), O._sinusoid_freqs(64, torch.float32).cuda(), B_SEED)

    # ------------------------------------------------------------------ FiLM generator (models/ncsn.py:47-61)
    if table_row is None and not mdn:
        R = 1 if bcast else batch
        tt = t.reshape(-1)[:R].to(F64)
        enc = v.f32("enc", R, 128)
        arg = F.noise_arg_f32(tt, v.f32("freqs", 64))
        rep.rel("FiLM noise encoding -> enc", enc, torch.cat([torch.sin(arg), torch.cos(arg)], dim=1), B_SEED)
        rep.launch("noise_encoding")
        for k in range(K):
            fp = f"k{k}.film."
            pre = enc @ P(fp + "d1.kernel") + P(fp + "d1.bias")
            if save:
                rep.rel(f"FiLM d1[{k}] pre-activation -> t.e1pre{k}", v.f32(f"t.e1pre{k}", R, 512), pre, B_DW)
            e1 = v.f32(f"t.e1_{k}", R, 512)
            rep.rel(f"FiLM d1[{k}] + swish -> t.e1_{k}", e1, F.swish(pre), B_DW)
            rep.launch(f"film d1[{k}]")
            e2 = v.f32(f"t.e2_{k}", R, 512)
            rep.rel(f"FiLM d2[{k}] -> t.e2_{k}", e2, e1 @ P(fp + "d2.kernel") + P(fp + "d2.bias"), B_DW)
            rep.launch(f"film d2[{k}]")
            ss = v.f32("ss", K, Bmax, 2 * Md)[k, :R]
            rep.rel(f"FiLM ss[{k}] -> ss", ss, e2 @ P(fp + "ss.kernel") + P(fp + "ss.bias"), B_DW)
            rep.launch(f"film ss[{k}]")

    # ------------------------------------------------------------------ trunk
    if dense:
        Cp = _ceil(Cc, 64)
        xb = v.b16("xb", M, Cp)[:, :Cc]
        rep.rel("cast x -> xb", xb, F.bf16_round(xin), B_EXACT)
        rep.launch("cast_bf16")
        u0 = v.f32("t.u0", M, Md)
        rep.rel("in GEMM -> t.u0", u0, F.gemm(xb, W("in.kernel"), P("in.bias"))["v"], B_DW)
        rep.launch("in gemm")
        if tangent:
            xbt = v.b16("xbt", M, Cp)[:, :Cc]
            rep.rel("tangent in GEMM -> t.ut0", v.f32("t.ut0", M, Md), xbt @ W("in.kernel"), B_DW)
            rep.launch("tangent in gemm")
    else:
        fused_attn = not save and S <= 64 and H in (8, 16) and not mdn
        fused_ffn = not save and M >= 32 * 256 and Md % 128 == 0
        h0, a = v.f32("t.h0", M, 128), v.b16("t.a1_0", M, 128)
        posenc = v.f32("posenc", S, 128)
        # float32 arguments s * f_j from the frequency table checked above, as the plan forms them; sin / cos in float64
        pos_arg = (torch.arange(S, dtype=torch.float32, device="cuda")[:, None] * v.raw("freqs", (64,), torch.float32)[None, :])
        pos_arg = pos_arg.to(F64)
        rep.rel("positional table posenc", posenc, torch.cat([torch.sin(pos_arg), torch.cos(pos_arg)], dim=1), B_SEED)
        h_ref, _ = F.embed(xin.reshape(batch, S, Cc), P("in.kernel"), P("in.bias"), posenc,
                           P("l0.ln1.scale"), P("l0.ln1.bias"))
        variant = "smem" if Cc <= 64 else "generic"
        rep.rel(f"embed ({variant}) -> t.h0", h0, h_ref.reshape(M, 128), B_DW)
        ref = F.layer_norm(h0, P("l0.ln1.scale"), P("l0.ln1.bias"))
        rep.bf16(f"embed ({variant}) LayerNorm -> t.a1_0", a, ref)
        rep.launch("embed")
        dh = 128 // H
        tf32 = dh % 8 == 0 and dh <= 32
        for l in range(Lt):
            pre = f"l{l}."
            nxt = f"l{l + 1}.ln1." if l + 1 < Lt else "post_ln."
            a_next_name = f"t.a1_{l + 1}" if l + 1 < Lt else "t.a_post"
            ln2 = (P(pre + "ln2.scale"), P(pre + "ln2.bias"))
            lnn = (P(nxt + "scale"), P(nxt + "bias"))
            a1, h_in = v.b16(f"t.a1_{l}", M, 128), v.f32(f"t.h{2 * l}", M, 128)
            h_mid, a2 = v.f32(f"t.h{2 * l + 1}", M, 128), v.b16(f"t.a2_{l}", M, 128)
            if fused_attn:
                ref, _ = F.attn_block(a1.reshape(batch, S, 128), h_in.reshape(batch, S, 128), W(pre + "attn.qkv.kernel"),
                                      P(pre + "attn.qkv.bias"), W(pre + "attn.out.kernel"), P(pre + "attn.out.bias"),
                                      *ln2, H)
                rep.rel(f"fused attention block[{l}] -> t.h{2 * l + 1}", h_mid, ref.reshape(M, 128), B_ATTN_BLOCK)
                ref = F.layer_norm(h_mid, *ln2)
                rep.bf16(f"fused attention block[{l}] LN2 -> t.a2_{l}", a2, ref)
                rep.launch(f"attn_block[{l}]")
            else:
                qkv = v.f32(f"t.qkv{l}", M, 384)
                rep.rel(f"QKV GEMM[{l}] -> t.qkv{l}", qkv, F.gemm(a1, W(pre + "attn.qkv.kernel"),
                                                                  P(pre + "attn.qkv.bias"))["v"], B_DW)
                rep.launch(f"qkv gemm[{l}]")
                probs_ref, o_ref = F.attention(qkv.reshape(batch, S, 384), H, causal=mdn)
                o = v.b16(f"t.o{l}", M, 128)
                kind = ("causal " if mdn else "") + ("tf32 mma" if tf32 else "SIMT")
                if tf32:
                    rep.rel(f"attention[{l}] ({kind}, dh {dh}) -> t.o{l}", o, o_ref.reshape(M, 128), B_TF32)
                else:
                    rep.bf16(f"attention[{l}] ({kind}, dh {dh}) -> t.o{l}", o, o_ref.reshape(M, 128))
                if save:
                    probs = v.f32(f"t.probs{l}", batch, H, S, S)
                    rep.rel(f"attention[{l}] probabilities -> t.probs{l}", probs, probs_ref, B_TF32 if tf32 else B_SEED)
                    rep.rel(f"attention[{l}] probability rows sum to 1", probs.sum(-1), torch.ones_like(probs[..., 0]),
                            B_SEED)
                    if mdn:
                        rep.zero(f"attention[{l}] probabilities above the diagonal (exact zeros)",
                                 probs * torch.ones(S, S, dtype=F64, device=probs.device).triu(1))
                rep.launch(f"attention[{l}]")
                e = F.gemm(o, W(pre + "attn.out.kernel"), P(pre + "attn.out.bias"), residual=h_in)
                rep.rel(f"out-proj[{l}] + residual -> t.h{2 * l + 1}", h_mid, e["v"], B_DW)
                ref = F.layer_norm(h_mid, *ln2)
                rep.bf16(f"out-proj[{l}] LN2 epilogue -> t.a2_{l}", a2, ref)
                rep.launch(f"out gemm[{l}]")
            h_out, a_next = v.f32(f"t.h{2 * l + 2}", M, 128), v.b16(a_next_name, M, 128)
            if fused_ffn:
                ref, _ = F.ffn_fused(a2, h_mid, W(pre + "ffn1.kernel"), P(pre + "ffn1.bias"), W(pre + "ffn2.kernel"),
                                     P(pre + "ffn2.bias"), *lnn)
                rep.rel(f"fused FFN[{l}] -> t.h{2 * l + 2}", h_out, ref, B_FFN_FUSED)
                ref = F.layer_norm(h_out, *lnn)
                rep.bf16(f"fused FFN[{l}] next LN -> {a_next_name}", a_next, ref)
                rep.launch(f"ffn_fused[{l}]")
                continue
            up = F.gemm(a2, W(pre + "ffn1.kernel"), P(pre + "ffn1.bias"), act="gelu")
            hid = v.b16(f"t.hid{l}", M, Md)
            rep.act(f"FFN-up[{l}] + GELU -> t.hid{l}", hid, up["act"], up["v"])
            if save:
                rep.bf16(f"FFN-up[{l}] pre-activation -> t.hpre{l}", v.b16(f"t.hpre{l}", M, Md), up["v"])
            rep.launch(f"ffn1 gemm[{l}]")
            e = F.gemm(hid, W(pre + "ffn2.kernel"), P(pre + "ffn2.bias"), residual=h_mid)
            rep.rel(f"FFN-down[{l}] + residual -> t.h{2 * l + 2}", h_out, e["v"], B_DW)
            ref = F.layer_norm(h_out, *lnn)
            rep.bf16(f"FFN-down[{l}] next LN epilogue -> {a_next_name}", a_next, ref)
            rep.launch(f"ffn2 gemm[{l}]")
        u0 = v.f32("t.u0", M, Md)
        rep.rel("post GEMM -> t.u0", u0, F.gemm(v.b16("t.a_post", M, 128), W("post.kernel"), P("post.bias"))["v"], B_DW)
        rep.launch("post gemm")

    # ------------------------------------------------------------------ FiLM'd residual tail
    if table_row is not None:
        T = eng._sampler_T
        tab = v.f32("ftab", K, T, 2 * Md)

    def rows_of(k):
        if mdn:   # TransformerMDN's res-blocks have no FiLM
            return None
        if table_row is not None:
            return F.film_rows(tab[k], M, S, row=table_row)
        return F.film_rows(v.f32("ss", K, Bmax, 2 * Md)[k, :(1 if bcast else batch)], M, S, broadcast=bcast)

    film_kind = "no" if mdn else ("table row" if table_row is not None else ("broadcast" if bcast else "per-example"))
    for k in range(K):
        pre = f"k{k}.res."
        rows = rows_of(k)
        u = v.f32(f"t.u{k}", M, Md)
        st = stats_all[2 * k]
        rep.rel(f"ln_film_act a[{k}] sums the partials of the GEMM before it -> stats[{2 * k}]", st, F.row_stats(u),
                B_SEED)
        ref, z = F.ln_film_act(u, st, P(pre + "ln_a.scale"), P(pre + "ln_a.bias"), rows, True)
        acta = v.b16(f"t.acta{k}", M, Md)
        rep.act(f"ln_film_act a[{k}] ({film_kind} FiLM) -> t.acta{k}", acta, ref, z)
        rep.launch(f"ln_film_act a[{k}]")
        if tangent:
            ut = v.f32(f"t.ut{k}", M, Md)
            actt = v.b16(f"t.actt{2 * k}", M, Md)
            rep.bf16(f"tangent ln_a[{k}] -> t.actt{2 * k}", actt,
                     F.ln_film_tangent(u, st, ut, P(pre + "ln_a.scale"), P(pre + "ln_a.bias"), rows, True))
            rep.launch(f"ln_film_tangent a[{k}]")
        e = F.gemm(acta, W(pre + "a.kernel"), P(pre + "a.bias"))
        r1 = v.b16(f"t.r1_{k}", M, Md)
        rep.bf16(f"res-a[{k}] -> t.r1_{k}", r1, e["v"])
        rep.launch(f"res-a gemm[{k}]")
        if tangent:
            r1t = v.f32(f"t.r1t{k}", M, Md)
            rep.rel(f"tangent res-a[{k}] -> t.r1t{k}", r1t, actt @ W(pre + "a.kernel"), B_DW)
            rep.launch(f"tangent res-a gemm[{k}]")
        st1 = stats_all[2 * k + 1]
        rep.rel(f"ln_film_act b[{k}] sums the res-a[{k}] epilogue partials -> stats[{2 * k + 1}]", st1, e["stats"], B_DW)
        ref, z = F.ln_film_act(r1, st1, P(pre + "ln_b.scale"), P(pre + "ln_b.bias"), rows, True)
        actb = v.b16(f"t.actb{k}", M, Md)
        rep.act(f"ln_film_act b[{k}] (bf16 input) -> t.actb{k}", actb, ref, z)
        rep.launch(f"ln_film_act b[{k}]")
        if tangent:
            acttb = v.b16(f"t.actt{2 * k + 1}", M, Md)
            rep.bf16(f"tangent ln_b[{k}] -> t.actt{2 * k + 1}", acttb,
                     F.ln_film_tangent(r1, st1, r1t, P(pre + "ln_b.scale"), P(pre + "ln_b.bias"), rows, True))
            rep.launch(f"ln_film_tangent b[{k}]")
        u1 = v.f32(f"t.u{k + 1}", M, Md)
        rep.rel(f"res-b[{k}] + residual -> t.u{k + 1}", u1, F.gemm(actb, W(pre + "b.kernel"), P(pre + "b.bias"),
                                                                    residual=u)["v"], B_DW)
        rep.launch(f"res-b gemm[{k}]")
        if tangent:
            rep.rel(f"tangent res-b[{k}] + residual -> t.ut{k + 1}", v.f32(f"t.ut{k + 1}", M, Md),
                    acttb @ W(pre + "b.kernel") + ut, B_DW)
            rep.launch(f"tangent res-b gemm[{k}]")
    uK = v.f32(f"t.u{K}", M, Md)
    st = stats_all[2 * K]
    rep.rel(f"ln_film_act out sums the res-b[{K - 1}] epilogue partials -> stats[{2 * K}]", st, F.row_stats(uK), B_SEED)
    act_out = v.b16("t.act_out", M, Md)
    ref, _ = F.ln_film_act(uK, st, P("out_ln.scale"), P("out_ln.bias"), None, False)
    rep.bf16("out_ln -> t.act_out", act_out, ref)
    rep.launch("ln_film_act out")
    if mdn:
        # the three head kernels packed into [Md][Hp] = [mu | log_sigma | pi], each part padded to 64 columns
        kc = cfg.mdn_components
        KCp, Kcp = _ceil(kc * Cc, 64), _ceil(kc, 64)
        Hp = 2 * KCp + Kcp
        w_head, b_head = v.b16("w.out_pad", Md, Hp), v.f32("mdn.head_bias", Hp)
        w_ref, b_ref = torch.zeros_like(w_head), torch.zeros_like(b_head)
        for pre, off, cols in (("mdn.mu.", 0, kc * Cc), ("mdn.log_sigma.", KCp, kc * Cc), ("mdn.pi.", 2 * KCp, kc)):
            w_ref[:, off:off + cols] = F.bf16_round(P(pre + "kernel"))
            b_ref[off:off + cols] = P(pre + "bias")
        rep.exact("packed head weight w.out_pad = bf16(mu | log_sigma | pi kernels), zero padding", w_head, w_ref)
        rep.exact("packed head bias mdn.head_bias", b_head, b_ref)
        rep.rel(f"head GEMM + head bias (N {Hp}) -> mdn.head", v.f32("mdn.head", M, Hp), act_out @ w_head + b_head, B_DW)
        rep.launch("head gemm")
        return v
    Hp = _ceil(Cc, 64)
    w_out = v.b16("w.out_pad", Md, Hp)[:, :Cc]
    rep.exact("padded output weight w.out_pad = bf16(out.kernel)", w_out, F.bf16_round(P("out.kernel")))
    rep.rel(f"out GEMM (N {Cc} of {Hp}) -> y", y.reshape(M, Cc).to(F64), act_out @ w_out + P("out.bias"), B_DW)
    rep.launch("out gemm")
    if tangent:
        acttK = v.b16(f"t.actt{2 * K}", M, Md)
        rep.bf16(f"tangent out_ln -> t.actt{2 * K}", acttK,
                 F.ln_film_tangent(uK, st, v.f32(f"t.ut{K}", M, Md), P("out_ln.scale"), P("out_ln.bias"), None, False))
        rep.launch("ln_film_tangent out")
        rep.rel("tangent out GEMM -> yt", v.f32("yt", M, Cc), acttK @ w_out, B_DW)
        rep.launch("tangent out gemm")
    return v


# ----------------------------------------------------------------------------------------------------------------------
# calls
# ----------------------------------------------------------------------------------------------------------------------
def _engine(arch, kw, max_batch, seed=2, **ekw):
    from smd_b200 import Engine, ModelConfig
    eng = Engine(ModelConfig(arch=arch, **kw), max_batch=max_batch, training=True, **ekw)
    eng.set_params(eng.init_params(seed=seed, perturb=0.05))
    return eng


def _inputs(batch, shape, seed):
    rng = np.random.default_rng(seed)
    x = rng.uniform(-1, 1, (batch, *shape)).astype(np.float32)
    t = rng.uniform(0.05, 1.0, (batch,)).astype(np.float32)
    return torch.from_numpy(x).cuda(), torch.from_numpy(t).cuda()


def _counted(eng, fn):
    torch.cuda.synchronize()
    n0 = eng.launch_count()
    out = fn()
    torch.cuda.synchronize()
    return out, eng.launch_count() - n0


def _infer(eng, x, t, bcast=False):
    """smd_forward (the inference path) on the training plan; bcast: t holds one value for every example."""
    y = torch.empty_like(x)
    L.check(eng.lib.smd_forward(eng._plan, eng.params.data_ptr(), x.data_ptr(), t.data_ptr(), 1 if bcast else 0,
                                x.shape[0], y.data_ptr(), torch.cuda.current_stream().cuda_stream))
    return y


def _save(eng, x, t):
    """The training forward (save = true): unfused kernels, probabilities and pre-activations kept."""
    y = torch.empty_like(x)
    L.check(eng.lib.smd_debug_forward_save(eng._plan, eng.params.data_ptr(), x.data_ptr(), t.data_ptr(), x.shape[0],
                                           y.data_ptr(), torch.cuda.current_stream().cuda_stream))
    return y


def _quiet_row0(d, layers):
    """Parameters under which position 0 of every sample keeps a row variance of about 1e-4 through the trunk's residual
    stream: in.bias cancels posenc[0] = [0]*64 + [1]*64 exactly, and in.kernel, the attention out-projection and the
    FFN down-projection are scaled by 1e-2.  On such rows LayerNorm's eps (1e-6) is about 1 % of the variance, and
    E[x^2] - E[x]^2 is formed from small sums."""
    d["in.bias"][:] = np.concatenate([np.zeros(64), -np.ones(64)]).astype(np.float32)
    d["in.kernel"] *= np.float32(0.015)
    for l in range(layers):
        for name in ("attn.out.kernel", "attn.out.bias", "ffn2.kernel", "ffn2.bias"):
            d[f"l{l}.{name}"] *= np.float32(0.01)


def run_case(name, arch, kw, batch, modes=("infer", "save"), bcast=False, seed=2, shift_film=None, quiet_row0=False):
    eng = _engine(arch, kw, batch, seed=seed)
    if quiet_row0:
        d = eng.flat_to_dict(eng.params.cpu().numpy().copy())
        _quiet_row0(d, eng.cfg.num_layers)
        eng.set_params(eng.dict_to_flat(d))
    if shift_film is not None:
        flat, Md = eng.params.cpu().numpy().copy(), eng.cfg.mlp_dims
        d = eng.flat_to_dict(flat)
        rng = np.random.default_rng(3)
        K = eng.cfg.num_layers if arch.startswith("Dense") else eng.cfg.num_mlp_layers
        for k in range(K):
            d[f"k{k}.film.ss.bias"][Md:] = rng.uniform(*shift_film, Md).astype(np.float32)
        eng.set_params(eng.dict_to_flat(d))
    shape = (kw.get("seq_len", 32), kw["channels"]) if arch.startswith("Transformer") else (kw["channels"],)
    x, t = _inputs(batch, shape, seed=21)
    if bcast:
        t = t[:1].contiguous()
    for mode in modes:
        rep = Report(f"{name} {mode}", (FAR_SHIFT, NOT_NEAREST_SHIFT) if shift_film else (BW.FAR, BW.NOT_NEAREST))
        if mode == "infer":
            y, n = _counted(eng, lambda: _infer(eng, x, t, bcast))
        else:
            y, n = _counted(eng, lambda: _save(eng, x, t))
        check_forward(eng, rep, x, t, batch, save=mode == "save", bcast=bcast, y=y)
        rep.expect_launches(n)
        rep.finish()
    return eng


T_KW = dict(num_layers=2, num_heads=8, num_mlp_layers=2, channels=42)
CASES = {
    # name: (arch, ModelConfig kwargs, batch, run_case options)
    # fused attention block with a half-filled last 64-row tile; the training-save forward on the same plan
    "L2_H8_K2_C42_b3": ("TransformerDDPM", T_KW, 3, {}),
    "S64_H16_b3": ("TransformerDDPM", dict(num_layers=1, num_heads=16, num_mlp_layers=1, channels=42, seq_len=64), 3, {}),
    "H4_b3": ("TransformerDDPM", dict(num_layers=1, num_heads=4, num_mlp_layers=1, channels=42), 3, {}),     # tf32, dh 32
    "H32_b3": ("TransformerDDPM", dict(num_layers=1, num_heads=32, num_mlp_layers=1, channels=42), 3, {}),   # SIMT, dh 4
    # head dim 8 at S 32 (the large model): attn_block_kernel<8, 32> and the tf32 training-save attention
    "H16_b3": ("TransformerDDPM", dict(num_layers=1, num_heads=16, num_mlp_layers=1, channels=42), 3, {}),
    "S128_H16_b2": ("TransformerDDPM", dict(num_layers=1, num_heads=16, num_mlp_layers=1, channels=42, seq_len=128), 2,
                    {}),
    # generic embed, output N 146 of 192, 1024-thread ln_film_act
    "C146_Md4096_b2": ("TransformerDDPM", dict(num_layers=1, num_heads=8, num_mlp_layers=1, channels=146,
                                               mlp_dims=4096), 2, {}),
    "Md256_b3": ("TransformerDDPM", dict(num_layers=1, num_heads=8, num_mlp_layers=2, channels=42, mlp_dims=256), 3, {}),
    "bcast_t_b1": ("TransformerDDPM", dict(num_layers=1, num_heads=8, num_mlp_layers=2, channels=42), 1,
                   dict(bcast=True, modes=("infer",))),
    "bcast_t_b3": ("TransformerDDPM", dict(num_layers=1, num_heads=8, num_mlp_layers=2, channels=42), 3,
                   dict(bcast=True, modes=("infer",))),
    # row 0 of every sample with a variance of about 1e-4 in the trunk (LayerNorm eps and variance on quiet rows)
    "quiet_row0_b3": ("TransformerDDPM", T_KW, 3, dict(quiet_row0=True)),
    "quiet_row0_b259": ("TransformerDDPM", dict(num_layers=1, num_heads=8, num_mlp_layers=1, channels=42), 259,
                        dict(quiet_row0=True, modes=("infer",))),
    # nearly every swish input of the tail in [-12, -3]
    "film_shift_negative": ("TransformerDDPM", dict(num_layers=1, num_heads=8, num_mlp_layers=2, channels=42), 3,
                            dict(shift_film=(-10.0, -5.0))),
    "dense_C512_b8": ("DenseDDPM", dict(num_layers=2, channels=512), 8, {}),
    "dense_C512_b130": ("DenseDDPM", dict(num_layers=2, channels=512), 130, {}),
}


@pytest.mark.parametrize("case", list(CASES))
def test_every_forward_launch_matches_its_fp64_restatement(lib, case):
    arch, kw, batch, opts = CASES[case]
    run_case(case, arch, kw, batch, **opts)


@pytest.mark.parametrize("batch", [259, 600])
def test_fused_ffn_and_attention_block_at_many_tiles(lib, batch):
    """259 samples: 8288 tokens, a partial last 128-row tile of the fused FFN; 600: 150 FFN tiles and 300 attention
    tiles, more than the SMs of an H100, so the persistent kernels loop over tiles."""
    run_case(f"fused_b{batch}", "TransformerDDPM", dict(num_layers=1, num_heads=8, num_mlp_layers=1, channels=42), batch,
             modes=("infer",))


def test_benchmarked_shape(lib):
    """L6/H8/K2/C42 at batch 128 (4096 tokens): overlap and wide GEMM layouts, statistics partials over 8 n-tiles."""
    run_case("base_b128", "TransformerDDPM", dict(num_layers=6, num_heads=8, num_mlp_layers=2, channels=42), 128)


def test_training_forward_inside_a_replayed_train_step_graph(lib):
    """The third compute_grads call on a capturable stream replays the captured train step: its saved activations obey
    the same rules as those of an eager training-save forward on the same plan."""
    arch, kw, batch = "TransformerDDPM", T_KW, 6
    eng = _engine(arch, kw, batch)
    eng.init_train_state()
    x, t = _inputs(batch, (32, 42), seed=23)
    rep = Report("graph eager save")
    y, n = _counted(eng, lambda: _save(eng, x, t))
    check_forward(eng, rep, x, t, batch, save=True, y=y)
    rep.expect_launches(n)
    rep.finish()
    eager = len(rep.launches)
    stream = torch.cuda.Stream()
    for step in range(3):
        x0, used, eps = BW._draws(batch, (32, 42), seed=60 + step)
        with torch.cuda.stream(stream):
            eng.compute_grads(x0, used, eps)
        torch.cuda.synchronize()
    v = BW.PlanView(eng)
    xt, tv = v.f32("xt", batch, 32, 42).float(), v.f32("tvec", batch).float()
    rep = Report("graph replay save")
    check_forward(eng, rep, xt, tv, batch, save=True, y=v.f32("eps_hat", batch, 32, 42))
    print(f"[parity] graph replay save: rules covered {len(rep.launches)} launches, eager training forward {eager}")
    assert len(rep.launches) == eager
    rep.finish()


def test_sampler_film_table_and_table_rows(lib):
    """A training plan with sampler_T = 1000: the FiLM table (gather + generator on all T conditioning values), one
    eager reverse step reading table row t, and one graph-replayed step reading the row through the device step
    counter (film_row_dev)."""
    check_sampler_step(_engine("TransformerDDPM", T_KW, 3, sampler_T=1000), 3, "sampler")


def check_sampler_step(eng, n, name, shard=None, inference_plan=False):
    """The rules of the DDPM sampler on a training plan with sampler_T = 1000, for n samples: the FiLM table, one eager
    reverse step at t = 500 with supplied noise (every forward launch, the step itself), then one graph-replayed step
    that must equal an eager step at t = T - 1 bit for bit.  shard: (first_row, total_rows) of set_sampler_shard.
    inference_plan: an inference plan of max_batch n (the one sample_ncsn and bench.py run) must replay the same step
    to the same bits as this training plan."""
    S, Cc = eng.seq_len, eng.cfg.channels
    betas = O.create_noise_schedule(1e-6, 0.01, 1000, "linear")
    eng.sampler_setup(betas, key=(0, 1))
    if shard is not None:
        eng.set_sampler_shard(*shard)
    x, _ = _inputs(n, (S, Cc), seed=24)
    z = torch.from_numpy(np.random.default_rng(25).standard_normal((n, S, Cc)).astype(np.float32)).cuda()
    eh = torch.empty_like(x)
    x_next, cnt = _counted(eng, lambda: eng.reverse_step(x, 500, z=z, eps_hat=eh))
    rep = Report(f"{name} eager step t=500")
    v = BW.PlanView(eng)
    K, Md, T = eng.cfg.num_mlp_layers, eng.cfg.mlp_dims, 1000
    # ---- the table: gather of the conditioning values, then the generator over all T rows
    tv = v.f32("ftab.t", T)
    rep.exact("FiLM table conditioning values ftab.t = coef[:, 5]", tv, v.f32("coef", T, 8)[:, 5])
    rep.launch("gather_cond")
    enc = v.f32("ftab.enc", T, 128)
    arg = F.noise_arg_f32(tv, v.f32("freqs", 64))
    rep.rel("FiLM table noise encoding -> ftab.enc", enc, torch.cat([torch.sin(arg), torch.cos(arg)], dim=1), B_SEED)
    rep.launch("table noise_encoding")
    tab = v.f32("ftab", K, T, 2 * Md)
    for k in range(K):
        fp = f"k{k}.film."
        e1 = F.swish(enc @ v.param(fp + "d1.kernel") + v.param(fp + "d1.bias"))
        e2 = e1 @ v.param(fp + "d2.kernel") + v.param(fp + "d2.bias")
        if k == K - 1:   # the generator's scratch rows hold the block that ran last
            rep.rel(f"FiLM table d1[{k}] -> ftab.e1", v.f32("ftab.e1", T, 512), e1, B_DW)
            rep.rel(f"FiLM table d2[{k}] -> ftab.e2", v.f32("ftab.e2", T, 512), e2, B_DW)
        rep.rel(f"FiLM table block {k}, all {T} rows -> ftab[{k}]", tab[k],
                e2 @ v.param(fp + "ss.kernel") + v.param(fp + "ss.bias"), B_DW)
        for part in ("d1", "d2", "ss"):
            rep.launch(f"table {part}[{k}]")
    t0 = time.perf_counter()
    check_forward(eng, rep, x, None, n, save=False, y=eh, table_row=500)
    print(f"[parity] {name}: float64 restatement of the forward of {n * S} tokens took "
          f"{time.perf_counter() - t0:.1f} s")
    coef = O.reverse_coefficients(betas)
    ref, _, _ = O.reverse_step(lambda s, c: eh.to(F64), x.to(F64), 500, coef, z.to(F64))
    rep.rel("reverse step -> x_next", x_next, ref, B_SEED)
    rep.launch("reverse_step")
    rep.expect_launches(cnt)
    rep.finish()
    # ---- graph: the step counter starts at T - 1 and is read on the device
    x2 = x.clone()
    _, cnt = _counted(eng, lambda: eng.sample(x2, steps=1, use_graph=True))
    rep = Report(f"{name} replayed step t=999")
    graph_eh = v.f32("eps_hat", n, S, Cc).clone()
    v = check_forward(eng, rep, x, None, n, save=False, y=graph_eh, table_row=T - 1)
    rep.exact("step_advance: device step counter", v.raw("t_ptr", (1,), torch.int32).to(F64),
              torch.tensor([T - 2], dtype=F64, device="cuda"))
    rep.launch("step_advance")
    # The replayed step draws its noise from threefry inside the graph.  An eager step at t = T - 1 without supplied
    # noise draws the same stream from the same key table, and its arithmetic is that of the step checked against the
    # oracle above: the replayed step must equal it bit for bit.
    eh2 = torch.empty_like(x)
    x_eager = eng.reverse_step(x, T - 1, eps_hat=eh2)
    torch.cuda.synchronize()
    rep.exact("replayed step network output = eager step's (table row T - 1)", graph_eh, eh2)
    rep.exact("replayed reverse step x_next = eager step at t = T - 1 (same threefry keys)", x2, x_eager)
    rep.launch("reverse_step (threefry noise)")
    rep.expect_launches(cnt)
    rep.finish()
    if not inference_plan:
        return
    # ---- the inference plan of the same model: the rules above read a training plan's buffers; the chains run here
    from smd_b200 import Engine
    inf = Engine(eng.cfg, max_batch=n, training=False)
    inf.set_params(eng.params)
    inf.sampler_setup(betas, key=(0, 1))
    if shard is not None:
        inf.set_sampler_shard(*shard)
    x3 = x.clone()
    inf.sample(x3, steps=1, use_graph=True)
    torch.cuda.synchronize()
    rep = Report(f"{name} inference plan")
    rep.exact("replayed step x_next on an inference plan = on the training plan", x3, x2)
    rep.finish()
    del inf


def test_dense_ncsn_tangent_pass_and_output_scale(lib):
    """DenseNCSN: the sliced score matching forward (q_sample, tangent cast, primal + tangent pass, loss), then an
    inference call on the same noised input whose raw output is that of the first call: the final division by sigma
    is checked exactly."""
    batch, Cc = 9, 64
    eng = _engine("DenseNCSN", dict(num_layers=2, channels=Cc), batch, seed=4)
    rng = np.random.default_rng(7)
    sigmas = O.create_noise_schedule(1.0, 0.01, 15, "geometric")
    x0, eps = (torch.from_numpy(rng.uniform(-1, 1, (batch, Cc)).astype(np.float32)).cuda(),
               torch.from_numpy(rng.standard_normal((batch, Cc)).astype(np.float32)).cuda())
    vv = torch.from_numpy(np.where(rng.random((batch, Cc)) < 0.5, 1.0, -1.0).astype(np.float32)).cuda()
    sig = torch.from_numpy(sigmas[rng.integers(0, 15, batch)].astype(np.float32)).cuda()
    (loss, score, hvp), cnt = _counted(eng, lambda: eng.ssm_loss(x0, sig, eps, vv, want_terms=True))
    rep = Report("ncsn ssm forward")
    v = BW.PlanView(eng)
    xt = v.f32("xt", batch, Cc)
    rep.rel("q_sample -> xt", xt, x0.to(F64) + sig.to(F64)[:, None] * eps.to(F64), B_SEED)
    rep.exact("q_sample -> conditioning sigma", v.f32("tvec", batch), sig)
    rep.launch("q_sample")
    rep.exact("tangent cast -> xbt", v.b16("xbt", batch, Cc), F.bf16_round(vv.to(F64)))
    rep.launch("tangent_input")
    f = v.f32("eps_hat", batch, Cc).clone()
    check_forward(eng, rep, xt.float(), sig, batch, save=False, y=f, tangent=True)
    ft, s64, v64 = v.f32("yt", batch, Cc), sig.to(F64), vv.to(F64)
    rep.rel("ssm loss -> loss", loss, 0.5 * (f * f).sum(1) + s64 * (v64 * ft).sum(1), B_SEED)
    rep.rel("ssm loss -> score", score, f / s64[:, None], B_SEED)
    rep.rel("ssm loss -> v.J v", hvp, (v64 * ft).sum(1) / s64, B_SEED)
    rep.launch("ssm_loss")
    rep.expect_launches(cnt)
    rep.finish()
    act_out = v.b16("t.act_out", batch, eng.cfg.mlp_dims).clone()
    xt32 = xt.float().contiguous()
    y, cnt = _counted(eng, lambda: eng.forward(xt32, sig))
    rep = Report("ncsn forward")
    check_forward(eng, rep, xt32, sig, batch, save=False, y=f)
    rep.exact("output layer input as in the ssm call", v.b16("t.act_out", batch, eng.cfg.mlp_dims), act_out)
    rep.exact("scale_rows: y = raw / sigma (fp32 division)", y, (f.float() / sig[:, None]))
    rep.launch("scale_rows")
    rep.expect_launches(cnt)
    rep.finish()


def test_transformer_mdn_causal_trunk_and_packed_head(lib):
    """TransformerMDN L2 H8: causal attention (tf32 mma) with and without saved probabilities, res-blocks without FiLM,
    and the head GEMM over the packed [mu | log_sigma | pi] weight with its packed bias.  The inference call is
    smd_mdn_forward without the input shift; the training-save forward is the first part of compute_mdn_grads, whose
    shift launch is checked too (its backward launches are test_gpu_backward_stages.py's)."""
    from smd_b200 import Engine, ModelConfig
    kw = dict(num_layers=2, num_heads=8, num_mlp_layers=2, channels=42, mdn_components=10)
    batch = 3
    eng = Engine(ModelConfig(arch="TransformerMDN", **kw), max_batch=batch, training=True)
    eng.set_params(eng.init_params(seed=2, perturb=0.05))
    eng.init_train_state()
    x = torch.from_numpy(np.random.default_rng(8).uniform(-1, 1, (batch, 32, 42)).astype(np.float32)).cuda()
    rep = Report("mdn infer")
    _, n = _counted(eng, lambda: eng.mdn_forward(x, shift=False))
    check_forward(eng, rep, x, None, batch, save=False)
    rep.expect_launches(n)
    rep.finish()
    infer_launches = len(rep.launches)
    eng.compute_mdn_grads(x)
    torch.cuda.synchronize()
    rep = Report("mdn save")
    v = BW.PlanView(eng)
    xs = v.f32("xt", batch, 32, 42)
    shifted = torch.cat([torch.zeros_like(x[:, :1]), x[:, :-1]], dim=1)
    rep.exact("input shift -> xt", xs, shifted)
    rep.launch("mdn_shift")
    check_forward(eng, rep, xs.float(), None, batch, save=True)
    # the training-save forward of TransformerMDN runs the inference call's launches (it has no fused path to leave)
    print(f"[parity] mdn save: rules covered {len(rep.launches)} launches, inference call {infer_launches} + shift")
    assert len(rep.launches) == infer_launches + 1
    rep.finish()
