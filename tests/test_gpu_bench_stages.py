"""Every launch of the workloads bench.py times, at the shapes it times them, against a float64 restatement of that
launch on the operands the device read.

Which kernel a launch runs depends on its shape (gemm_kind and expand_groups in csrc/gemm_host.cuh, the attention
backward's head-count dispatch, the embedding's channel-count dispatch), so the rules of test_gpu_forward_stages.py and
test_gpu_backward_stages.py are run here at the benchmarked shapes and no others:

- cfg4 (L8/H16/K3, C 42) and c512 (L6/H8/K2, C 512), trained at batch 128 per GPU: the training-save and the inference
  forward, then the device draws and the gradient call of an 8-GPU global batch (1024 examples), then the optimizer
  step.  Head dim 8 at S 32, the output GEMM at N 512, the global-memory embedding and its chunked backward.
- the reverse step of cfg3 / cfg5 at 1000 samples (32 000 tokens, C 42 and C 146), the strong-scaling shards of 500,
  250 and 125 samples as the last rank of 2, 4 and 8, and 125 samples on a plan that has just run 1000 (rows [M, Mp)
  of every activation hold the larger call's values).  The rules read a training plan's buffers; the benchmark samples
  on an inference plan, so at 1000 and 125 samples an inference plan must replay the same step to the same bits.
- the bf16 weight shadow every tensor-core GEMM reads (wshadow).  The stage rules restate each GEMM from the shadow the
  device read, so a stale or wrongly rounded shadow is invisible to them: here it is compared bit for bit with the
  round-to-nearest bf16 of the fp32 parameters after set_params, after every optimizer step (clip_adam_kernel writes
  it), on the kernel's vector body, its scalar tail and its all-scalar unaligned path, and on the engines the nn.Model
  path of train_ncsn re-packs through a version tag.

The optimizer rules restate clip_adam_kernel's fp32 formula in float64 from the device's inputs and from the clip
factor the device derived from its own sum of squares: the constants are the fp32 values the kernel holds (1 - beta2
is 0.000999987 in fp32, 1.3e-5 away from 0.001), so every difference left is one fp32 rounding per operation (B_SEED).

Bounds are those of the two stage files; no new one is needed.  Each test prints its wall time and the peak device
memory torch allocated (the plan's workspace included), and the sampler tests print how long the float64 restatement
of one forward took and the workspace of the plan.

Measured on an H100 80GB HBM3 (SXM, 700 W power limit):

- largest errors of the optimizer rules: sum of squares 9.5e-8, m / v / p / EMA 8.6e-8 (B_SEED 4e-7); the shadow and
  w.out_pad differ from bf16_rn of the parameters in no element after set_params and after every step
- the float64 restatement of the forward of 32 000 tokens through six layers: 0.3 s
- a training plan of max_batch 1000, sampler_T 1000: 6.0 GiB of workspace; the 1000-sample test peaks at 14.4 GiB
  with the inference plan and the float64 references; every test of this file finishes within 6 s
"""
import gc
import math
import time

import numpy as np
import pytest
import torch

from oracle import ddpm_oracle as O
from smd_b200 import lib as L
from tests import test_gpu_backward_stages as BW
from tests import test_gpu_forward_stages as FW

pytestmark = pytest.mark.gpu

F64 = torch.float64
B_SEED = BW.B_SEED
BASE = dict(num_layers=6, num_heads=8, num_mlp_layers=2)
LARGE = dict(num_layers=8, num_heads=16, num_mlp_layers=3)
BATCH, GLOBAL_BATCH = 128, 1024       # bench.py: 128 examples per GPU, 8 GPUs
BETAS = O.create_noise_schedule(1e-6, 0.01, 1000, "linear")


@pytest.fixture(autouse=True)
def _wall_and_peak_memory(request):
    gc.collect()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    yield
    torch.cuda.synchronize()
    print(f"[parity] {request.node.name}: wall {time.perf_counter() - t0:.1f} s, peak device memory "
          f"{torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB")
    gc.collect()
    torch.cuda.empty_cache()


# ----------------------------------------------------------------------------------------------------------------------
# the bf16 weight shadow and the optimizer step
# ----------------------------------------------------------------------------------------------------------------------
def _bitwise(rep, rule, got, ref):
    """Two bf16 tensors with the same bits (so that -0 and +0 differ)."""
    assert got.shape == ref.shape, (rule, got.shape, ref.shape)
    n = int((got.contiguous().view(torch.int16) != ref.contiguous().view(torch.int16)).sum())
    print(f"[parity] {rep.case} {rule}: differing bits in {n}/{ref.numel()}{'' if n == 0 else '  <-- FAILED'}")
    rep.rules += 1
    if n:
        rep.failed.append((rule, n, 0))


def shadow_rules(eng, rep, params=None, engine=""):
    """wshadow = bf16_rn(params) over the whole arena, and the padded output weight w.out_pad = bf16_rn(out.kernel) with
    zero pad columns.  params: the fp32 arena the engine's next forward reads (default: the engine's own); engine: a
    name for the engine in the rule names."""
    torch.cuda.synchronize()
    params = eng.params if params is None else params
    v = BW.PlanView(eng)
    n = eng.arena_floats
    _bitwise(rep, f"{engine}wshadow = bf16_rn(parameter arena)", v.raw("wshadow", (n,), torch.bfloat16),
             params.to(torch.bfloat16))
    Md, Cc = eng.cfg.mlp_dims, eng.cfg.channels
    Hp = BW._ceil(Cc, 64)
    off, shape = v.layout["out.kernel"]
    ref = torch.zeros((Md, Hp), dtype=torch.bfloat16, device=params.device)
    ref[:, :Cc] = params[off:off + Md * Cc].reshape(shape).to(torch.bfloat16)
    _bitwise(rep, f"{engine}w.out_pad = bf16_rn(out.kernel), pad columns {Cc}..{Hp} zero",
             v.raw("w.out_pad", (Md, Hp), torch.bfloat16), ref)


def adam_rules(rep, before, after, total, gnorm, *, step, lr, max_norm, b1=0.9, b2=0.999, eps=1e-8, mu=0.999):
    """sumsq_kernel + clip_adam_kernel: before = {p, g, m, v[, ema]} as the launch read them, after = {p, m, v[, ema]}
    as it wrote them; total = scratch[0] and gnorm = the post-clip norm it stored."""
    f32 = lambda a: float(np.float32(a))  # noqa: E731  (the value the kernel holds)
    B1, B2, LR, EPS, MU, MAXN = f32(b1), f32(b2), f32(lr), f32(eps), f32(mu), f32(max_norm)
    bc1, bc2 = f32(1.0 - B1 ** (step + 1.0)), f32(1.0 - B2 ** (step + 1.0))   # formed in double on the host
    g = before["g"].to(F64)
    total = total.reshape(1).to(F64)
    rep.rel("sumsq partials summed in clip_adam -> scratch[0]", total, (g * g).sum().reshape(1), B_SEED)
    norm = math.sqrt(float(total))                  # the clip factor from the device's own total
    factor = 1.0 if norm < MAXN else MAXN / norm
    rep.rel(f"post-clip gradient norm -> grad_norm ({'clipped' if factor < 1 else 'not clipped'}: norm {norm:.3e}, "
            f"max {MAXN:.3e})", gnorm.reshape(1), torch.tensor([norm * factor], dtype=F64, device=g.device), B_SEED)
    gc_ = g * factor
    m = (1.0 - B1) * gc_ + B1 * before["m"].to(F64)   # 1 - B1 and 1 - B2 are exact in fp32 (Sterbenz)
    v = (1.0 - B2) * gc_ * gc_ + B2 * before["v"].to(F64)
    p = before["p"].to(F64) - LR * (m / bc1) / (torch.sqrt(v / bc2) + EPS)
    rep.rel("Adam first moment m", after["m"], m, B_SEED)
    rep.rel("Adam second moment v", after["v"], v, B_SEED)
    rep.rel("Adam parameters p", after["p"], p, B_SEED)
    if "ema" in before:
        ema = before["ema"].to(F64) * MU + after["p"].to(F64) * (1.0 - MU)
        rep.rel("EMA of the new parameters", after["ema"], ema, B_SEED)


def apply_grads_rules(eng, name, lr=1e-3, grad_clip=1.0):
    """Engine.apply_grads as train_step runs it: sumsq, clip_adam (which refreshes the shadow) and the re-pack of the
    padded output weight, three launches."""
    before = dict(p=eng.params.clone(), g=eng.grads.clone(), m=eng.adam_m.clone(), v=eng.adam_v.clone())
    step = eng.opt_step
    _, cnt = FW._counted(eng, lambda: eng.apply_grads(lr=lr, grad_clip=grad_clip))
    rep = FW.Report(f"{name} optimizer step {step}")
    adam_rules(rep, before, dict(p=eng.params, m=eng.adam_m, v=eng.adam_v), eng._scratch[0], eng.grad_norm,
               step=step, lr=lr, max_norm=grad_clip)
    rep.launch("sumsq")
    rep.launch("clip_adam")
    shadow_rules(eng, rep)
    rep.launch("pad_cast_bf16 out.kernel -> w.out_pad")
    rep.expect_launches(cnt)
    rep.finish()


# ----------------------------------------------------------------------------------------------------------------------
# train step at the benchmarked shapes
# ----------------------------------------------------------------------------------------------------------------------
def run_train_case(name, kw):
    from smd_b200 import Engine, ModelConfig
    eng = Engine(ModelConfig(arch="TransformerDDPM", **kw), max_batch=BATCH, training=True)
    flat = eng.init_params(seed=2, perturb=0.05)
    _, cnt = FW._counted(eng, lambda: eng.set_params(flat))
    rep = FW.Report(f"{name} set_params")
    shadow_rules(eng, rep)
    rep.launch("cast_bf16 -> wshadow")
    rep.launch("pad_cast_bf16 out.kernel -> w.out_pad")
    rep.expect_launches(cnt)
    rep.finish()
    eng.init_train_state()
    eng.objective_setup(BETAS)
    Cc = kw["channels"]
    x, t = FW._inputs(BATCH, (32, Cc), seed=21)
    for mode, call in (("save", FW._save), ("infer", FW._infer)):
        rep = FW.Report(f"{name} {mode}")
        y, cnt = FW._counted(eng, lambda: call(eng, x, t))
        FW.check_forward(eng, rep, x, t, BATCH, save=mode == "save", y=y)
        rep.expect_launches(cnt)
        rep.finish()
    # the draws of rank 0 of an 8-GPU global batch, as bench.py's train step makes them
    x0 = torch.from_numpy(np.random.default_rng(22).uniform(-1, 1, (BATCH, 32, Cc)).astype(np.float32)).cuda()
    used, eps = eng.draws((3, 17), BATCH, global_batch=GLOBAL_BATCH)
    eng.compute_grads(x0, used, eps, global_batch=GLOBAL_BATCH)
    rep = BW.check_stages(eng, BATCH, FW.Report(f"{name} backward"), eps=eps, global_batch=GLOBAL_BATCH)
    BW.assert_complete(eng, rep)
    rep.finish()
    apply_grads_rules(eng, name)


def test_cfg4_large_train_step_at_batch128(lib):
    """L8/H16/K3, C 42: head dim 8 at S 32 (attn_block_kernel<8, 32>, the tf32 training-save attention and its
    backward), three res-blocks, 4096 tokens."""
    run_train_case("cfg4_b128", dict(channels=42, **LARGE))


def test_c512_train_step_at_batch128(lib):
    """L6/H8/K2, C 512: the output GEMM at N 512 (8-warp kEpiF32), its dX at K 512 over 512 tiles, its dW at N 512, the
    global-memory embedding (C > 64) and its backward over 8 channel chunks, the loss seed on 512 columns."""
    run_train_case("c512_b128", dict(channels=512, **BASE))


# ----------------------------------------------------------------------------------------------------------------------
# the optimizer kernel on its three paths
# ----------------------------------------------------------------------------------------------------------------------
PAD = 64          # floats (or bf16) of sentinel on each side of every arena
SENTINEL = 7.25   # no parameter, moment, EMA or shadow value of these cases comes near it

CLIP_ADAM_CASES = {
    # name: (n, offset of every arena in elements, step, gradient scale)
    "unaligned_all_scalar": ((1 << 20) + 4, 1, 0, 3e-3),   # vec_ok = 0: every element on the scalar path
    "n_1_mod_4": ((1 << 20) + 1, 0, 3, 3e-3),              # vector body + a scalar tail of 1, clipped
    "n_2_mod_4": ((1 << 20) + 2, 0, 0, 5e-4),              # ... of 2, not clipped
    "n_3_mod_4": ((1 << 20) + 3, 0, 7, 3e-3),              # ... of 3, clipped, with moments from earlier steps
}


def _fenced(vals, off, dtype=torch.float32):
    """(buffer, view): vals at element PAD + off of a sentinel-filled buffer."""
    n = vals.numel()
    buf = torch.full((n + 2 * PAD,), SENTINEL, dtype=dtype, device="cuda")
    view = buf[PAD + off:PAD + off + n]
    view.copy_(vals.to(dtype))
    return buf, view


@pytest.mark.parametrize("case", list(CLIP_ADAM_CASES))
def test_clip_adam_paths_and_shadow(lib, case):
    """smd_clip_adam on arenas fenced by sentinels: m, v, p, EMA and the bf16 shadow of every element in [0, n), and
    nothing written outside it."""
    n, off, step, scale = CLIP_ADAM_CASES[case]
    rng = np.random.default_rng(40 + step)
    dev = lambda a: torch.from_numpy(np.asarray(a, np.float32)).cuda()   # noqa: E731
    p0 = dev(rng.standard_normal(n) * 0.05)
    init = dict(p=p0, g=dev(rng.standard_normal(n) * scale),
                m=dev(rng.standard_normal(n) * 1e-4) if step else torch.zeros_like(p0),
                v=dev(rng.random(n) * 1e-7) if step else torch.zeros_like(p0),
                ema=p0 + dev(rng.standard_normal(n) * 1e-3))
    bufs, views = {}, {}
    for k, a in init.items():
        bufs[k], views[k] = _fenced(a, off)
    bufs["shadow"], views["shadow"] = _fenced(torch.zeros(n, device="cuda"), off, torch.bfloat16)
    before = {k: a.clone() for k, a in init.items()}
    scratch, gnorm = torch.zeros(1024, device="cuda"), torch.zeros(1, device="cuda")
    lr, max_norm = 1e-3, 1.0
    torch.cuda.synchronize()
    n0 = lib.smd_launch_count()
    L.check(lib.smd_clip_adam(*(views[k].data_ptr() for k in ("p", "g", "m", "v", "ema", "shadow")), n, lr, step,
                              max_norm, 0.9, 0.999, 1e-8, 0.999, scratch.data_ptr(), gnorm.data_ptr(),
                              torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    cnt = lib.smd_launch_count() - n0
    rep = FW.Report(f"clip_adam {case} (n = {n}, offset {off}, step {step})")
    adam_rules(rep, before, views, scratch[0], gnorm, step=step, lr=lr, max_norm=max_norm)
    rep.launch("sumsq")
    _bitwise(rep, "shadow = bf16_rn(p)", views["shadow"], views["p"].to(torch.bfloat16))
    rep.launch("clip_adam")
    for k, buf in bufs.items():
        outside = torch.cat([buf[:PAD + off], buf[PAD + off + n:]])
        rep.zero(f"{k}: elements outside [0, n) changed", (outside != SENTINEL).to(torch.int32))
    rep.exact("g is read only", views["g"], before["g"])
    rep.expect_launches(cnt)
    rep.finish()


def _bf16_moved(rep, rule, before_bits, flat, least=0.01):
    """The step changed bf16_rn of at least `least` of the arena's elements: a shadow left from before the step would
    differ from the one the rules demand, so the shadow rules can see a missed re-pack."""
    n = int((flat.to(torch.bfloat16).view(torch.int16) != before_bits).sum())
    share = n / flat.numel()
    ok = share >= least
    print(f"[parity] {rep.case} {rule}: bf16_rn changed in {n}/{flat.numel()} elements ({share:.3f}, at least "
          f"{least}){'' if ok else '  <-- FAILED'}")
    rep.rules += 1
    if not ok:
        rep.failed.append((rule, share, least))


def test_optimizer_on_the_model_path_refreshes_every_engine_shadow(lib):
    """train_ncsn.train_step through nn.Model and optim.Adam, with three engines that each serve one arena:

    - the training engine, whose parameters alias the model's arena: clip_adam writes its shadow in the step;
    - the model's cached inference engine of max_batch 3: only the arena version bump of optim.Optimizer makes it
      re-pack (its tag holds the same arena object before and after the step);
    - the EMA model's inference engine, from a module of its own so that no other arena passes through it: only the
      bump of the EMA arena makes it re-pack.

    Each inference engine runs a forward, then the step, then its next forward, with nothing in between.  After each of
    two steps every engine reads a shadow equal to bf16_rn of its arena, and the step changed bf16_rn of both arenas
    in most elements (the EMA runs at mu = 0.5 so that one step moves it by more than a bf16 spacing)."""
    from absl import flags

    from smd_b200 import jrandom as random
    from smd_b200 import ncsn, nn, optim, train_ncsn, train_utils
    from smd_b200.losses import diffusion_loss
    if not flags.FLAGS.is_parsed():
        flags.FLAGS.mark_as_parsed()
    B = 8
    kw = dict(num_layers=1, num_heads=8, num_mlp_layers=1, mlp_dims=2048)
    module, ema_module = ncsn.TransformerDDPM.partial(**kw), ncsn.TransformerDDPM.partial(**kw)
    # a one-example init: the module caches only an inference engine of max_batch 1, which no call below fits in
    _, params = module.init_by_shape(random.PRNGKey(0), [((1, 32, 42), np.float32), ((1, 1, 1), np.float32)])
    model = nn.Model(module, params)
    optimizer = optim.Adam().create(model)
    ema = train_utils.EMAHelper(0.5, model.arena.clone())
    ema_model = nn.Model(ema_module, ema.params)
    rng = np.random.default_rng(9)
    x = rng.uniform(-1, 1, (B, 32, 42)).astype(np.float32)
    t = rng.uniform(0.05, 1.0, (B, 1, 1)).astype(np.float32)
    model(x[:3], t[:3])
    ema_model(x[:5], t[:5])
    inf_eng, ema_eng = model.engine(3), ema_model.engine(5)
    assert inf_eng.max_batch == 3 and ema_eng.max_batch == 5 and not inf_eng.training and not ema_eng.training
    assert all(e is not ema_eng for e in module._engines) and all(e is not inf_eng for e in ema_module._engines)
    mu = flags.FLAGS.mu
    flags.FLAGS.mu = ema.mu
    try:
        for step in range(2):
            model_bits = model.arena.flat.to(torch.bfloat16).view(torch.int16)
            ema_bits = ema.params.flat.to(torch.bfloat16).view(torch.int16)
            optimizer, _ = train_ncsn.train_step(diffusion_loss, x, optimizer, BETAS,
                                                 np.array([0, 30 + step], np.uint32), 1e-3, ema)
            rep = FW.Report(f"nn.Model path after step {step}")
            _bf16_moved(rep, "the step moved the model arena", model_bits, model.arena.flat)
            _bf16_moved(rep, "the step moved the EMA arena", ema_bits, ema.params.flat)
            train_eng = model.engine(B, training=True)
            assert train_eng.params.data_ptr() == model.arena.flat.data_ptr()   # the aliasing clip_adam relies on
            train_eng.forward(torch.from_numpy(x).cuda(), torch.from_numpy(t).cuda().reshape(-1))
            shadow_rules(train_eng, rep, model.arena.flat, "training engine: ")
            model(x[:3], t[:3])
            assert model.engine(3) is inf_eng
            shadow_rules(inf_eng, rep, model.arena.flat, "inference engine (max_batch 3): ")
            ema_model(x[:5], t[:5])
            assert ema_model.engine(5) is ema_eng
            shadow_rules(ema_eng, rep, ema.params.flat, "EMA engine (max_batch 5): ")
            rep.finish()
    finally:
        flags.FLAGS.mu = mu


# ----------------------------------------------------------------------------------------------------------------------
# reverse step at the benchmarked sample counts
# ----------------------------------------------------------------------------------------------------------------------
def _sampler_engine(channels, max_batch):
    eng = FW._engine("TransformerDDPM", dict(channels=channels, **BASE), max_batch, sampler_T=1000)
    print(f"[parity] training plan max_batch {max_batch}, sampler_T 1000, C {channels}: workspace "
          f"{eng.workspace_bytes / 2 ** 30:.2f} GiB")
    return eng


@pytest.mark.parametrize("channels", [42, 146])
def test_reverse_step_at_1000_samples(lib, channels):
    """cfg3 / cfg5: 32 000 tokens, the fused FFN and attention block over more tiles than SMs, the expand kernel over
    250 row blocks, at C 146 the output GEMM over 500 tiles; sharded as bench.py's single-GPU job, (0, 1000)."""
    FW.check_sampler_step(_sampler_engine(channels, 1000), 1000, f"n1000_c{channels}", shard=(0, 1000),
                          inference_plan=channels == 42)


@pytest.mark.parametrize("world", [2, 4, 8])
def test_reverse_step_strong_scaling_shard(lib, world):
    """1000 // world samples on a plan of that size, as the last rank of a sharded chain.  125 samples (4000 tokens)
    leave a partial last 128-row block and run the FFN unfused."""
    n = 1000 // world
    FW.check_sampler_step(_sampler_engine(42, n), n, f"shard{world - 1}of{world}_n{n}",
                          shard=((world - 1) * n, n * world), inference_plan=n == 125)


def test_reverse_step_125_samples_after_1000_on_the_same_plan(lib):
    """Rows [4000, 4096) of every activation still hold the 1000-sample call's values."""
    eng = _sampler_engine(42, 1000)
    eng.sampler_setup(BETAS, key=(0, 1))
    x = torch.from_numpy(np.random.default_rng(26).standard_normal((1000, 32, 42)).astype(np.float32)).cuda()
    eng.reverse_step(x, 700, z=torch.randn_like(x))
    torch.cuda.synchronize()
    FW.check_sampler_step(eng, 125, "n125_after_n1000")
