"""Backward / optimizer parity: hand-written CUDA backward vs torch autograd on the CPU oracle.

Tolerances (stated): per-tensor rel-L2 <= 3e-2 for tensors carrying >= 1e-4 of the gradient energy, global cosine
>= 0.9995 and |norm ratio - 1| <= 1e-2 (bf16 tensor-core operands in both forward and backward GEMMs; at the benchmarked
sizes tests/test_gpu_bench_shapes.py asserts tighter bounds -- the small batches here are noisier per tensor)."""
import numpy as np
import pytest
import torch

from oracle import ddpm_oracle as O
from tests.util import oracle_kwargs, params_torch, rel_l2

pytestmark = pytest.mark.gpu

CASES = {
    "tiny": (dict(num_layers=1, num_heads=8, num_mlp_layers=1, channels=42), "TransformerDDPM", 4),
    "base2": (dict(num_layers=2, num_heads=8, num_mlp_layers=2, channels=42), "TransformerDDPM", 6),
    "large_h16": (dict(num_layers=2, num_heads=16, num_mlp_layers=3, channels=146), "TransformerDDPM", 3),
    "dense": (dict(num_layers=2, channels=512), "DenseDDPM", 8),
    "heads4": (dict(num_layers=1, num_heads=4, num_mlp_layers=1, channels=42), "TransformerDDPM", 3),
    "heads32": (dict(num_layers=1, num_heads=32, num_mlp_layers=1, channels=42), "TransformerDDPM", 3),
}


def _draws(batch, shape, seed=0):
    rng = np.random.default_rng(seed)
    x0 = rng.uniform(-1, 1, (batch, *shape)).astype(np.float32)
    eps = rng.standard_normal((batch, *shape)).astype(np.float32)
    betas = O.create_noise_schedule(1e-6, 0.01, 1000, "linear")
    ap = O.alphas_prod_with_one(betas)
    labels = rng.integers(1, 1001, size=batch)
    return x0, ap[labels - 1].astype(np.float32), eps


def _oracle_grads(arch, eng, flat, x0, used, eps, emulate):
    p = {k: v.clone().requires_grad_(True) for k, v in params_torch(eng, flat).items()}
    okw = oracle_kwargs(eng.cfg)
    loss, _ = O.diffusion_loss_tensors(lambda a, c: O.model_apply(arch, p, a, c, emulate_bf16=emulate, **okw),
                                       torch.from_numpy(x0), torch.from_numpy(used), torch.from_numpy(eps), "mean")
    loss.backward()
    return float(loss), {k: (v.grad if v.grad is not None else torch.zeros_like(v)) for k, v in p.items()}


@pytest.mark.parametrize("cg", [1, 2])
@pytest.mark.parametrize("case", list(CASES))
def test_gradients_match_autograd(lib, case, cg):
    from smd_b200 import Engine, ModelConfig
    kw, arch, batch = CASES[case]
    cfg = ModelConfig(arch=arch, **kw)
    eng = Engine(cfg, max_batch=batch, cta_group=cg, training=True)
    flat = eng.init_params(seed=2, perturb=0.05)
    eng.set_params(flat)
    eng.init_train_state()
    shape = (32, kw["channels"]) if arch != "DenseDDPM" else (kw["channels"],)
    x0, used, eps = _draws(batch, shape)
    eng.compute_grads(torch.from_numpy(x0).cuda(), torch.from_numpy(used).cuda(), torch.from_numpy(eps).cuda())
    torch.cuda.synchronize()
    got = eng.flat_to_dict(eng.grads)
    loss_ref, ref = _oracle_grads(arch, eng, flat, x0, used, eps, emulate=False)
    assert abs(float(eng.loss_sum) / batch - loss_ref) < 5e-3 * loss_ref
    total = sum(float((g ** 2).sum()) for g in ref.values())
    dot = nn_got = 0.0
    report = []
    for name, g in ref.items():
        gg = torch.from_numpy(got[name])
        dot += float((gg * g).sum())
        nn_got += float((gg ** 2).sum())
        e = rel_l2(gg, g)
        report.append((e, name))
        if float((g ** 2).sum()) >= 1e-4 * total:
            assert e < 3e-2, f"{name}: rel-L2 {e:.3e}\n" + "\n".join(f"{a:.3e} {b}" for a, b in sorted(report)[-12:])
    cos = dot / (np.sqrt(nn_got) * np.sqrt(total))
    assert cos > 0.9995, (cos, sorted(report)[-12:])
    assert abs(np.sqrt(nn_got / total) - 1.0) < 1e-2
    # every tensor (also the tiny ones) must at least be close in absolute terms
    for name, g in ref.items():
        gg = torch.from_numpy(got[name])
        assert float((gg - g).abs().max()) < 5e-2 * float(np.sqrt(total / max(1, len(ref)))) + 1e-6, name


def test_clip_adam_matches_flax_restatement(lib):
    from smd_b200 import Engine, ModelConfig
    eng = Engine(ModelConfig(num_layers=1, num_mlp_layers=1), max_batch=2, training=True)
    flat = eng.init_params(seed=3, perturb=0.05)
    eng.set_params(flat)
    eng.init_train_state(ema=True)
    rng = np.random.default_rng(0)
    for scale in (1e-4, 3e-3):   # un-clipped and clipped (norm > 1)
        g = (rng.standard_normal(eng.arena_floats) * scale).astype(np.float32)
        p0 = eng.params.cpu().clone(); m0 = eng.adam_m.cpu().clone(); v0 = eng.adam_v.cpu().clone()
        e0 = eng.ema_params.cpu().clone()
        eng.grads.copy_(torch.from_numpy(g))
        step = eng.opt_step
        eng.apply_grads(lr=1e-3, grad_clip=1.0)
        torch.cuda.synchronize()
        gt = torch.from_numpy(g)
        norm = float(gt.double().norm())
        gc = gt if norm < 1.0 else gt * (1.0 / norm)
        p1, m1, v1 = O.adam_step(p0, gc, m0, v0, step, 1e-3)
        assert abs(float(eng.grad_norm) - min(norm, 1.0)) < 1e-4 * max(1.0, norm)
        assert rel_l2(eng.adam_m, m1) < 1e-5 and rel_l2(eng.adam_v, v1) < 1e-4
        assert float((eng.params.cpu() - p1).abs().max()) < 2e-6
        assert rel_l2(eng.ema_params, O.ema_update(e0, p1, 0.999)) < 1e-6


def test_train_steps_reduce_loss_and_track_oracle(lib):
    """Three optimizer steps on a fixed batch: loss / grad-norm / update direction follow the oracle's train_step."""
    from smd_b200 import Engine, ModelConfig
    kw = dict(num_layers=1, num_heads=8, num_mlp_layers=1, channels=42)
    eng = Engine(ModelConfig(**kw), max_batch=8, cta_group=2, training=True)
    flat = eng.init_params(seed=5, perturb=0.02)
    eng.set_params(flat)
    eng.init_train_state()
    x0, used, eps = _draws(8, (32, 42), seed=4)
    args = [torch.from_numpy(a).cuda() for a in (x0, used, eps)]
    p = params_torch(eng, flat)
    m = {k: torch.zeros_like(v) for k, v in p.items()}
    v = {k: torch.zeros_like(t) for k, t in p.items()}
    losses = []
    for step in range(3):
        loss, gn = eng.train_step(*args, lr=1e-3)
        losses.append(float(loss))
        (p, m, v), oloss, ognorm, _ = O.train_step("TransformerDDPM", p, m, v, step, torch.from_numpy(x0),
                                                    torch.from_numpy(used), torch.from_numpy(eps), 1e-3,
                                                    model_kw=oracle_kwargs(eng.cfg))
        assert abs(losses[-1] - float(oloss)) < 3e-2 * float(oloss)
        assert abs(float(gn) - float(ognorm)) < 3e-2 * float(ognorm) + 1e-4
    got = eng.flat_to_dict(eng.params)
    # Adam's first steps move every weight by ~lr regardless of gradient scale: compare the update direction
    moved = agree = 0
    for k, t in p.items():
        d_ref = t - torch.from_numpy(eng.flat_to_dict(flat)[k])
        d_got = torch.from_numpy(got[k]) - torch.from_numpy(eng.flat_to_dict(flat)[k])
        moved += d_ref.numel()
        agree += int((torch.sign(d_ref) == torch.sign(d_got)).sum())
    assert agree / moved > 0.97


def test_device_draws_match_jax_restatement(lib):
    """labels / used_alpha / eps of diffusion_loss generated on device == the jax-0.2.8 threefry restatement."""
    from smd_b200 import Engine, ModelConfig
    from oracle import threefry as tf
    eng = Engine(ModelConfig(num_layers=1, num_mlp_layers=1), max_batch=64, training=False)
    eng.set_params(eng.init_params(0))
    betas = O.create_noise_schedule(1e-6, 0.01, 1000, "linear")
    eng.objective_setup(betas)
    for seed, batch in ((0, 64), (123, 7)):
        key = tf.prng_key(seed)
        used, eps, labels = eng.draws((int(key[0]), int(key[1])), batch, want_labels=True)
        rl, ru, re = O.diffusion_loss_draws(key, (batch, 32, 42), betas, continuous_noise=True)
        np.testing.assert_array_equal(labels.cpu().numpy(), rl)
        np.testing.assert_array_equal(used.cpu().numpy(), ru)           # == abar[l-1] (SURVEY D8)
        np.testing.assert_allclose(eps.cpu().numpy(), re, rtol=2e-5, atol=2e-6)


def test_tail_gradients_are_final_at_the_tail_event(lib):
    """smd_wait_tail_grads: a second stream that waits on it sees the final tail slice while the trunk backward is
    still in flight on the main stream (what the overlapped all-reduce relies on)."""
    import ctypes as C
    from smd_b200 import Engine, ModelConfig
    from smd_b200 import lib as L
    kw, arch, batch = CASES["base2"]
    eng = Engine(ModelConfig(arch=arch, **kw), max_batch=batch, cta_group=2, training=True)
    eng.set_params(eng.init_params(seed=2, perturb=0.05))
    eng.init_train_state()
    shape = (32, kw["channels"])
    x0, used, eps = _draws(batch, shape)
    first, count = eng.grads_tail_range()
    side = torch.cuda.Stream()
    snap = torch.empty(count, dtype=torch.float32, device="cuda")
    for _ in range(3):
        eng.compute_grads(torch.from_numpy(x0).cuda(), torch.from_numpy(used).cuda(), torch.from_numpy(eps).cuda())
        with torch.cuda.stream(side):
            L.check(eng.lib.smd_wait_tail_grads(eng._plan, C.c_void_p(side.cuda_stream)))
            snap.copy_(eng.grads[first:first + count], non_blocking=True)
        torch.cuda.synchronize()
        assert torch.equal(snap, eng.grads[first:first + count])
        assert float(eng.grads[:first].abs().sum()) > 0


def test_graph_replayed_step_equals_eager_launches(lib):
    """On a capturable stream smd_ddpm_grads replays one CUDA graph (3-stream fork / join captured once, per-step input
    pointers through a device table).  Same gradients as the eager launches, also when every step brings new tensors,
    and the tail-gradient events still work from a stream outside the graph."""
    import ctypes as C
    from smd_b200 import Engine, ModelConfig
    from smd_b200 import lib as L
    kw, arch, batch = CASES["base2"]
    shape = (32, kw["channels"])

    def make():
        e = Engine(ModelConfig(arch=arch, **kw), max_batch=batch, cta_group=2, training=True)
        e.set_params(e.init_params(seed=2, perturb=0.05))
        e.init_train_state()
        return e

    eager, graph = make(), make()
    stream, side = torch.cuda.Stream(), torch.cuda.Stream()
    first, count = graph.grads_tail_range()
    snap = torch.empty(count, dtype=torch.float32, device="cuda")
    for step in range(5):
        x0, used, eps = _draws(batch, shape, seed=10 + step)
        args = [torch.from_numpy(a).cuda() for a in (x0, used, eps)]       # fresh tensors every step
        eager.compute_grads(*args)                                         # legacy default stream: never captured
        torch.cuda.synchronize()
        n0 = graph.launch_count()
        with torch.cuda.stream(stream):
            graph.compute_grads(*[a.clone() for a in args])                # step 0 eager (warm-up), 1 captures, 2.. replay
            with torch.cuda.stream(side):
                L.check(graph.lib.smd_wait_tail_grads(graph._plan, C.c_void_p(side.cuda_stream)))
                snap.copy_(graph.grads[first:first + count], non_blocking=True)
        torch.cuda.synchronize()
        assert graph.launch_count() - n0 > 50                              # replayed launches are still counted
        assert rel_l2(graph.grads, eager.grads) < 1e-5, step               # (split-K atomics: not bitwise)
        assert torch.equal(snap, graph.grads[first:first + count]), step   # the tail slice was final at the event
        assert abs(float(graph.loss_sum) - float(eager.loss_sum)) <= 1e-6 * abs(float(eager.loss_sum))

