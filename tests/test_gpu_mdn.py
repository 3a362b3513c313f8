"""TransformerMDN (models/autoregressive.py, train_mdn.py) through the C ABI against the CPU restatement in
tests/mdn_reference.py: forward (causal trunk + mixture-density head), the mixture NLL, the loss and its gradients.

Tolerances are about twice the errors measured on an H100 with bf16 tensor-core operands."""
import ctypes
import os
import re
import subprocess
import sys
import textwrap

import numpy as np
import pytest
import torch

from tests import mdn_reference as R
from tests.util import params_torch, rel_l2

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KW = dict(num_layers=2, num_heads=8, num_mlp_layers=2, mlp_dims=2048, mdn_components=100)
C = 42


def _engine(batch, training=False, **over):
    from smd_b200 import Engine, ModelConfig
    kw = dict(KW, **over)
    eng = Engine(ModelConfig(arch="TransformerMDN", channels=C, **kw), max_batch=batch, training=training)
    flat = eng.init_params(seed=5, perturb=0.02)
    eng.set_params(flat)
    return eng, flat


def _x(B, seed):
    return np.random.default_rng(seed).uniform(-1, 1, (B, 32, C)).astype(np.float32)


def _ref(p, x, shift=True, emulate=False):
    return R.transformer_mdn(p, x, shift=shift, emulate_bf16=emulate, **KW)


# num_heads 8: the tf32 mma.sync causal kernel (head dim 16); 32: the SIMT causal kernel (head dim 4)
@pytest.mark.parametrize("shift,heads", [(True, 8), (False, 8), (True, 32)])
def test_forward_matches_oracle(lib, shift, heads):
    eng, flat = _engine(4, num_heads=heads)
    x = _x(4, 0)
    got = eng.mdn_forward(torch.from_numpy(x).cuda(), shift=shift)
    torch.cuda.synchronize()
    pe = params_torch(eng, flat, torch.float32)
    pd = params_torch(eng, flat, torch.float64)
    kw = dict(KW, num_heads=heads)
    tight = R.transformer_mdn(pe, torch.from_numpy(x), shift=shift, emulate_bf16=True, **kw)
    loose = R.transformer_mdn(pd, torch.from_numpy(x).double(), shift=shift, **kw)
    e_t = [rel_l2(g, r) for g, r in zip(got, tight)]
    e_l = [rel_l2(g, r) for g, r in zip(got, loose)]
    print(f"mdn forward shift={shift} heads={heads}: rel-L2 (pi, mu, log_sigma) vs bf16-emulating oracle {e_t}, vs fp64 {e_l}")
    assert max(e_t) < 1e-2 and max(e_l) < 3e-2


@pytest.mark.parametrize("heads", [8, 32])
def test_causality_on_device(lib, heads):
    eng, _ = _engine(2, num_heads=heads)
    x = torch.from_numpy(_x(2, 1)).cuda()
    base = eng.mdn_forward(x)
    for j in (0, 13, 31):
        x2 = x.clone()
        x2[:, j] += 0.5
        out = eng.mdn_forward(x2)
        for a, b in zip(base, out):
            # with the shift, position j's input first reaches the output at position j + 1
            assert torch.equal(a[:, :j + 1], b[:, :j + 1]), j
            if j + 1 < 32:
                assert not torch.equal(a[:, j + 1:], b[:, j + 1:]), j


def test_nll_matches_fp64(lib):
    from smd_b200 import load_library
    rng = np.random.default_rng(2)
    rows, kc = 300, 100
    pi = rng.normal(0, 3, (rows, kc)).astype(np.float32)
    mu = rng.normal(0, 1, (rows, kc * C)).astype(np.float32)
    ls = rng.uniform(-3, 1.5, (rows, kc * C)).astype(np.float32)   # sigma from 0.05 to 4.5
    x = rng.normal(0, 1, (rows, C)).astype(np.float32)
    d = [torch.from_numpy(a).cuda() for a in (pi, mu, ls, x)]
    loss = torch.empty(rows, device="cuda")
    lb = load_library()
    rc = lb.smd_mdn_nll(*[t.data_ptr() for t in d], rows, C, kc, loss.data_ptr(), torch.cuda.current_stream().cuda_stream)
    assert rc == 0
    torch.cuda.synchronize()
    ref = R.mdn_nll(*[torch.from_numpy(a).double() for a in (pi, mu, ls, x)])
    err = float(((loss.cpu().double() - ref).abs() / ref.abs().clamp_min(1.0)).max())
    print(f"mdn nll: max rel err {err:.3e}")
    assert err <= 1e-5


def test_loss_matches_oracle(lib):
    eng, flat = _engine(4)
    x = _x(4, 3)
    got = eng.mdn_loss(torch.from_numpy(x).cuda())
    torch.cuda.synchronize()
    pd = params_torch(eng, flat, torch.float64)
    xd = torch.from_numpy(x).double()
    ref = R.mdn_nll(*_ref(pd, xd), xd)
    err = rel_l2(got, ref)
    print(f"mdn loss: rel-L2 {err:.3e}, mean {float(got.mean()):.4f} vs {float(ref.mean()):.4f}")
    assert got.shape == (4 * 32,) and err < 1e-2


def test_grads_match_fp64_autograd(lib):
    B, GB = 4, 8
    eng, flat = _engine(B, training=True)
    eng.init_train_state()
    x = _x(B, 4)
    eng.compute_mdn_grads(torch.from_numpy(x).cuda(), global_batch=GB)
    torch.cuda.synchronize()
    p = {k: t.requires_grad_(True) for k, t in params_torch(eng, flat, torch.float64).items()}
    xd = torch.from_numpy(x).double()
    per = R.mdn_nll(*_ref(p, xd), xd)
    (per.sum() / (GB * 32)).backward()
    assert abs(float(eng.loss_sum) - float(per.sum())) < 1e-2 * abs(float(per.sum()))
    assert abs(float(eng.loss_mean) - float(per.sum()) / (GB * 32)) < 1e-2 * abs(float(per.sum()) / (GB * 32))
    got = eng.flat_to_dict(eng.grads)
    tot = sum(float((t.grad ** 2).sum()) for t in p.values())
    errs = {k: rel_l2(torch.from_numpy(got[k]), t.grad) for k, t in p.items() if float((t.grad ** 2).sum()) >= 1e-4 * tot}
    dot = sum(float((torch.from_numpy(got[k]).double() * t.grad).sum()) for k, t in p.items())
    nn_ = sum(float((torch.from_numpy(got[k]).double() ** 2).sum()) for k in p)
    cos = dot / np.sqrt(nn_ * tot)
    worst = max(errs.items(), key=lambda kv: kv[1])
    print(f"mdn grads: cos {cos:.6f}, worst tensor {worst}, mdn.* {[(k, round(v, 5)) for k, v in errs.items() if 'mdn' in k]}")
    # measured on an H100: cos 0.99843, worst tensor 6.4e-2 (in.kernel; the head's own 3e-2 .. 6e-2).  The mixture
    # responsibilities softmax(lp) amplify the bf16 forward error: lp is ~80 nats per token at this scale
    assert cos > 0.997 and worst[1] < 0.13, worst


def test_grads_are_reproducible_and_graph_replay_matches_eager(lib):
    eng, _ = _engine(8, training=True)
    eng.init_train_state()
    a = torch.from_numpy(_x(8, 5)).cuda()
    b = torch.from_numpy(_x(8, 6)).cuda()
    stream = torch.cuda.Stream()
    outs = []
    with torch.cuda.stream(stream):
        for inp in (a, a, a, b):        # eager (first use), capture + replay, replay, replay with a new tensor
            eng.compute_mdn_grads(inp)
            outs.append((eng.grads.clone(), eng.loss_sum.clone()))
    stream.synchronize()
    for g, l in outs[1:3]:
        torch.testing.assert_close(g, outs[0][0], rtol=1e-4, atol=1e-7)   # atomics ordering only
        assert torch.equal(l, outs[0][1])
    eng.compute_mdn_grads(b)            # legacy default stream: eager
    torch.cuda.synchronize()
    torch.testing.assert_close(outs[3][0], eng.grads, rtol=1e-4, atol=1e-7)
    assert torch.equal(outs[3][1], eng.loss_sum)
    l1, l2 = eng.mdn_loss(a), eng.mdn_loss(a)
    f1, f2 = eng.mdn_forward(a), eng.mdn_forward(a)
    assert torch.equal(l1, l2) and all(torch.equal(u, v) for u, v in zip(f1, f2))


def test_graph_replay_equals_eager_subprocess(lib, tmp_path):
    code = f"""
import sys, numpy as np, torch
sys.path.insert(0, {ROOT!r})
from tests.test_gpu_mdn import _engine, _x
eng, _ = _engine(8, training=True)
eng.init_train_state()
x = torch.from_numpy(_x(8, 7)).cuda()
s = torch.cuda.Stream()
with torch.cuda.stream(s):
    for _ in range(3):
        eng.compute_mdn_grads(x)
s.synchronize()
np.save(sys.argv[1], np.concatenate([eng.grads.cpu().numpy(), eng.loss_sum.cpu().numpy()]))
"""
    outs = []
    for flag in ("1", "0"):
        path = tmp_path / f"g{flag}.npy"
        r = subprocess.run([sys.executable, "-c", code, str(path)], env=dict(os.environ, SMD_TRAIN_GRAPH=flag),
                           capture_output=True, text=True, timeout=600, cwd=ROOT)
        assert r.returncode == 0, r.stderr[-3000:]
        outs.append(np.load(path))
    np.testing.assert_allclose(outs[0][:-1], outs[1][:-1], rtol=1e-4, atol=1e-7)
    assert outs[0][-1] == outs[1][-1]


def test_other_entry_points_reject_an_mdn_plan(lib):
    from smd_b200 import Engine, ModelConfig
    eng, _ = _engine(2, training=True)
    eng.init_train_state()
    x = torch.from_numpy(_x(2, 8)).cuda()
    t = torch.ones(2, device="cuda")
    with pytest.raises(ValueError):
        eng.forward(x, t)
    with pytest.raises(ValueError):
        eng.ddpm_loss(x, t, x)
    with pytest.raises(ValueError):
        eng.compute_grads(x, t, x)
    with pytest.raises(ValueError):
        eng.dsm_loss(x, t, x)
    with pytest.raises(ValueError):
        eng.sampler_setup(np.full(10, 0.01, np.float32))
    with pytest.raises(ValueError):
        eng.reverse_step(x, 0)
    with pytest.raises(ValueError):
        eng.sample(x, steps=1)
    with pytest.raises(ValueError):
        eng.mdn_forward(x[:, :, :C - 1].contiguous())     # channels must match the plan
    for over in (dict(seq_len=64), dict(seq_len=128), dict(mdn_components=0)):
        with pytest.raises(ValueError):
            Engine(ModelConfig(arch="TransformerMDN", channels=C, **dict(KW, **over)), max_batch=2)
    with pytest.raises(ValueError):
        Engine(ModelConfig(arch="TransformerMDN", channels=C, **KW), max_batch=2, precision="bf16x3")
    ddpm = Engine(ModelConfig(channels=C), max_batch=2)
    ddpm.set_params(ddpm.init_params(seed=0))
    assert ddpm.lib.smd_mdn_loss(ddpm._plan, ddpm.params.data_ptr(), x.data_ptr(), 2, x.data_ptr(), None) == -1


def test_training_lowers_the_loss(lib):
    eng, _ = _engine(16, training=True)
    eng.init_train_state()
    x = torch.from_numpy(_x(16, 9)).cuda()
    before = float(eng.mdn_loss(x).mean())
    for _ in range(10):
        eng.compute_mdn_grads(x)
        eng.apply_grads(3e-4)
    after = float(eng.mdn_loss(x).mean())
    print(f"mdn train: loss {before:.4f} -> {after:.4f}")
    assert np.isfinite(after) and after < before
    first, count = eng.grads_tail_range()
    names = [n for n, off, _ in eng.layout if off >= first]
    assert names[0] == "k0.res.ln_a.scale" and names[-1] == "mdn.pi.bias" and first + count == eng.arena_floats


def test_tail_gradients_are_final_at_the_event(lib):
    """smd_wait_tail_grads: the k*, out_ln and mdn.* slice is complete when the event fires (eager and replayed)."""
    from smd_b200 import lib as L
    eng, _ = _engine(8, training=True)
    eng.init_train_state()
    x = torch.from_numpy(_x(8, 11)).cuda()
    first, count = eng.grads_tail_range()
    stream, side = torch.cuda.Stream(), torch.cuda.Stream()
    snap = torch.empty(count, dtype=torch.float32, device="cuda")
    for _ in range(3):                                       # eager, capture + replay, replay
        with torch.cuda.stream(stream):
            eng.compute_mdn_grads(x)
            with torch.cuda.stream(side):
                L.check(eng.lib.smd_wait_tail_grads(eng._plan, ctypes.c_void_p(side.cuda_stream)))
                snap.copy_(eng.grads[first:first + count], non_blocking=True)
        torch.cuda.synchronize()
        assert torch.equal(snap, eng.grads[first:first + count])
        assert float(eng.grads[:first].abs().sum()) > 0


def test_train_mdn_cli_lowers_the_loss_and_checkpoints(tmp_path):
    cfg = tmp_path / "mdn.cfg"
    cfg.write_text(textwrap.dedent(f"""\
        --architecture=TransformerMDN
        --num_layers=2
        --num_heads=8
        --num_mlp_layers=2
        --mlp_dims=512
        --mdn_components=20
        --data_shape=32,42
        --batch_size=16
        --learning_rate=1e-3
        --logging_freq=1
        --snapshot_freq=10
        --nosnapshot_sampling
        --synthetic
        --synthetic_examples=640
        --model_dir={tmp_path / 'run'}
        """))
    env = dict(os.environ, PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, "-m", "smd_b200.train_mdn", f"--flagfile={cfg}", "--max_steps=20"],
                       capture_output=True, text=True, timeout=600, env=env, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-3000:]
    losses = [float(v) for v in re.findall(r"\] \[epoch \d+\] step \d+/\d+: loss=([-0-9.e+]+)", r.stderr)]
    print(f"train_mdn losses: {losses[:3]} ... {losses[-3:]}")
    assert len(losses) >= 20 and np.isfinite(losses).all() and np.mean(losses[-3:]) < np.mean(losses[:3])
    from smd_b200 import autoregressive as ar, checkpoints, nn, optim, train_utils
    names = checkpoints.list_checkpoints(str(tmp_path / "run"))
    assert names == ["checkpoint_0", "checkpoint_1"], names

    def template():
        module = ar.TransformerMDN.partial(num_layers=2, num_heads=8, num_mlp_layers=2, mlp_dims=512, mdn_mixtures=20)
        _, params = module.init_by_shape(None, [((16, 32, 42), np.float32)], seed=123)
        return optim.Adam(learning_rate=1e-3).create(nn.Model(module, params)), train_utils.EarlyStopping(patience=1)

    opt, es = checkpoints.restore_checkpoint(str(tmp_path / "run"), template())
    assert opt.step >= 20 and np.isfinite(es.best_metric)
    x = torch.from_numpy(_x(2, 12)).cuda()
    pi, mu, ls = opt.target(x)                                    # model(inputs) -> (pi, mu, log_sigma)
    assert pi.shape == (2, 32, 20) and mu.shape == ls.shape == (2, 32, 20 * 42)
    checkpoints.save_checkpoint(str(tmp_path / "flax"), (opt, es), 0, fmt="flax")
    opt2, es2 = checkpoints.restore_checkpoint(str(tmp_path / "flax"), template())
    assert torch.equal(opt2.target.arena.flat, opt.target.arena.flat) and opt2.step == opt.step
    assert torch.equal(opt2.grad_sq_ema, opt.grad_sq_ema) and es2.state_dict() == es.state_dict()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs >= 2 GPUs")
def test_dp_grads_equal_single_rank():
    w = min(torch.cuda.device_count(), 8)
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={w}",
                        "--master-addr", "127.0.0.1", "--master-port", "29541",
                        os.path.join(ROOT, "tests", "mdn_dp_worker.py")], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "mdn-dp-ok" in r.stdout, r.stdout[-2000:] + r.stderr[-3000:]
