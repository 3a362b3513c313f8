"""TransformerDDPM at sequence lengths 64 and 128: forward (fused attention block at S = 64, unfused path at S = 128),
strict mode, hand-written backward, saved attention probabilities, sampler and the train / sample command lines, each
against the CPU oracle with the tolerances of the S = 32 suites (test_gpu_forward, test_gpu_strict, test_gpu_train,
test_gpu_sampler, test_gpu_sharding)."""
import math
import os
import pickle
import subprocess
import sys
import textwrap

import numpy as np
import pytest
import torch

from oracle import ddpm_oracle as O
from oracle import threefry as tf
from tests.test_gpu_plan_buffers import _region
from tests.test_gpu_train import _draws, _oracle_grads
from tests.util import make_inputs, oracle_kwargs, params_torch, rel_l2

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
C = 42


def _kw(heads, layers=2, mlp_layers=1):
    return dict(num_layers=layers, num_heads=heads, num_mlp_layers=mlp_layers, channels=C)


def _engine(kw, S, batch, training=False, precision="bf16", seed=1, perturb=0.02):
    from smd_b200 import Engine, ModelConfig
    eng = Engine(ModelConfig(seq_len=S, **kw), max_batch=batch, cta_group=2, training=training, precision=precision)
    flat = eng.init_params(seed=seed, perturb=perturb)
    eng.set_params(flat)
    return eng, flat


def _check_forward(eng, flat, x, t):
    y = eng.forward(torch.from_numpy(x).cuda(), torch.from_numpy(t).cuda())
    torch.cuda.synchronize()
    okw = oracle_kwargs(eng.cfg)
    ref_bf = O.transformer_ddpm(params_torch(eng, flat), torch.from_numpy(x), torch.from_numpy(t), emulate_bf16=True, **okw)
    ref32 = O.transformer_ddpm(params_torch(eng, flat), torch.from_numpy(x), torch.from_numpy(t), **okw)
    ref64 = O.transformer_ddpm(params_torch(eng, flat, torch.float64), torch.from_numpy(x).double(),
                               torch.from_numpy(t).double(), **okw)
    assert rel_l2(y, ref_bf) < 1e-2
    assert rel_l2(y, ref32) < 1.2e-2 and rel_l2(y, ref64) < 1.2e-2
    assert float((y.cpu() - ref32).abs().max()) < 6e-2


# head dims 16 / 8 (mma attention, fused block at S = 64) and 32 / 4 (mma / SIMT attention, unfused)
@pytest.mark.parametrize("heads", [8, 16, 4, 32])
@pytest.mark.parametrize("S", [64, 128])
def test_forward_parity(lib, S, heads):
    eng, flat = _engine(_kw(heads), S, 3)
    x, t = make_inputs(7, 3, (S, C))
    _check_forward(eng, flat, x, t)


def test_forward_fused_ffn_batch_and_ragged_batch(lib):
    """S = 64, batch 128 = 8192 tokens: the fused FFN runs next to the fused attention block; batch 5 does not."""
    eng, flat = _engine(_kw(8, layers=1), 64, 128)
    for seed, batch in ((3, 128), (4, 5)):
        x, t = make_inputs(seed, batch, (64, C))
        _check_forward(eng, flat, x, t)


@pytest.mark.parametrize("S", [64, 128])
def test_strict_forward_matches_fp64_oracle(lib, S):
    eng, flat = _engine(_kw(8), S, 3, precision="bf16x3")
    x, t = make_inputs(7, 3, (S, C))
    y = eng.forward(torch.from_numpy(x).cuda(), torch.from_numpy(t).cuda())
    ref64 = O.transformer_ddpm(params_torch(eng, flat, torch.float64), torch.from_numpy(x).double(),
                               torch.from_numpy(t).double(), **oracle_kwargs(eng.cfg))
    assert rel_l2(y, ref64) < 1e-4


@pytest.mark.parametrize("S,heads", [(64, 8), (128, 8), (64, 4), (128, 16), (128, 32)])
def test_gradients_match_autograd(lib, S, heads):
    batch = 3
    eng, flat = _engine(_kw(heads, layers=1), S, batch, training=True, seed=2, perturb=0.05)
    eng.init_train_state()
    x0, used, eps = _draws(batch, (S, C))
    eng.compute_grads(torch.from_numpy(x0).cuda(), torch.from_numpy(used).cuda(), torch.from_numpy(eps).cuda())
    torch.cuda.synchronize()
    got = eng.flat_to_dict(eng.grads)
    loss_ref, ref = _oracle_grads("TransformerDDPM", eng, flat, x0, used, eps, emulate=False)
    assert abs(float(eng.loss_sum) / batch - loss_ref) < 5e-3 * loss_ref
    total = sum(float((g ** 2).sum()) for g in ref.values())
    for name, g in ref.items():
        if float((g ** 2).sum()) >= 1e-4 * total:
            e = rel_l2(torch.from_numpy(got[name]), g)
            assert e < 3e-2, (name, e)


def test_train_steps_track_oracle(lib):
    eng, flat = _engine(_kw(8, layers=1), 64, 4, training=True, seed=5)
    eng.init_train_state()
    x0, used, eps = _draws(4, (64, C), seed=4)
    args = [torch.from_numpy(a).cuda() for a in (x0, used, eps)]
    p = params_torch(eng, flat)
    m = {k: torch.zeros_like(v) for k, v in p.items()}
    v = {k: torch.zeros_like(t) for k, t in p.items()}
    for step in range(3):
        loss, gn = eng.train_step(*args, lr=1e-3)
        (p, m, v), oloss, ognorm, _ = O.train_step("TransformerDDPM", p, m, v, step, torch.from_numpy(x0),
                                                    torch.from_numpy(used), torch.from_numpy(eps), 1e-3,
                                                    model_kw=oracle_kwargs(eng.cfg))
        assert abs(float(loss) - float(oloss)) < 3e-2 * float(oloss)
        assert abs(float(gn) - float(ognorm)) < 3e-2 * float(ognorm) + 1e-4


def test_saved_probabilities_are_the_oracle_softmax(lib):
    """t.probs of a training forward at S = 128 holds softmax(q k^T / sqrt(dh)) as [B][H][S][S]."""
    from smd_b200 import lib as L
    S, H, batch = 128, 8, 2
    eng, flat = _engine(_kw(H, layers=1), S, batch, training=True)
    x, t = make_inputs(7, batch, (S, C))
    xd, td = torch.from_numpy(x).cuda(), torch.from_numpy(t).cuda()
    y = torch.empty_like(xd)
    L.check(eng.lib.smd_debug_forward_save(eng._plan, eng.params.data_ptr(), xd.data_ptr(), td.data_ptr(), batch,
                                           y.data_ptr(), torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    p = params_torch(eng, flat)
    trace = {}
    O.transformer_ddpm(p, torch.from_numpy(x), torch.from_numpy(t), emulate_bf16=True, trace=trace,
                       **oracle_kwargs(eng.cfg))
    a1 = trace["t.a1_0"].to(torch.bfloat16).float()
    qkv = O.dense(a1, p["l0.attn.qkv.kernel"], p["l0.attn.qkv.bias"], True)
    dh = 128 // H
    q, k, _ = qkv.split(128, dim=-1)
    q = q.reshape(batch, S, H, dh) / math.sqrt(dh)
    k = k.reshape(batch, S, H, dh)
    ref = torch.softmax(torch.einsum("bqhd,bkhd->bhqk", q, k), dim=-1)
    got = _region(eng, "t.probs0", (batch, H, S, S), torch.float32)
    assert rel_l2(got, ref) < 1e-2
    assert float((got.sum(-1) - 1).abs().max()) < 1e-4


def _sampler(S, batch, key=(0, 7)):
    eng, flat = _engine(_kw(8, layers=1), S, batch)
    betas = O.create_noise_schedule(1e-6, 0.01, 1000, "linear")
    eng.sampler_setup(betas, key=key)
    p = params_torch(eng, flat)
    okw = oracle_kwargs(eng.cfg)
    return eng, betas, lambda a, c: O.transformer_ddpm(p, a, c, emulate_bf16=True, **okw)


def test_reverse_step_supplied_noise(lib):
    eng, betas, apply_bf = _sampler(64, 4)
    rng = np.random.default_rng(1)
    x = torch.from_numpy(rng.standard_normal((4, 64, C)).astype(np.float32))
    z = torch.from_numpy(rng.standard_normal((4, 64, C)).astype(np.float32))
    eh = torch.empty((4, 64, C), device="cuda")
    nxt = eng.reverse_step(x.cuda(), 500, z=z.cuda(), eps_hat=eh)
    ref_next, ref_eps, _ = O.reverse_step(apply_bf, x, 500, O.reverse_coefficients(betas), z)
    assert rel_l2(eh, ref_eps) < 1e-2 and rel_l2(nxt, ref_next) < 1e-2


def test_graph_replayed_chain_matches_oracle(lib):
    key = (0, 7)
    eng, betas, apply_bf = _sampler(64, 4, key)
    init = torch.from_numpy(np.random.default_rng(0).standard_normal((4, 64, C)).astype(np.float32))
    x = init.clone().cuda()
    eng.sample(x, steps=4, use_graph=True)
    torch.cuda.synchronize()
    rkey = np.array(key, np.uint32)
    keys = []
    for _ in range(4):
        rkey, _unused = tf.split(rkey, 2)
        rkey, _infill = tf.split(rkey, 2)
        rkey, noise_k = tf.split(rkey, 2)
        keys.append(noise_k)
    ref, _, _ = O.diffusion_dynamics(apply_bf, betas, init,
                                     lambda i, t: (torch.from_numpy(tf.normal(keys[i], (4, 64, C))), None), steps=4)
    assert rel_l2(x, ref) < 1e-2


def test_sharded_sampling_equals_the_single_process_chain(lib):
    from smd_b200 import jrandom
    key, steps = (0, 21), 3
    one, betas, _ = _sampler(64, 8, key)
    init_key = jrandom.PRNGKey(3)
    ref = jrandom.normal(init_key, (8, 64, C))
    one.sample(ref, steps=steps, use_graph=True)
    for r in range(2):
        eng, _, _ = _sampler(64, 4, key)
        eng.set_sampler_shard(4 * r, 8)
        x = jrandom.normal(init_key, (8, 64, C), rows=(4 * r, 4))
        eng.sample(x, steps=steps, use_graph=(r == 0))
        assert torch.equal(x, ref[4 * r:4 * r + 4])


def test_train_and_sample_cli_at_64_latents(tmp_path):
    cfg = tmp_path / "ddpm-64seq.cfg"
    cfg.write_text(textwrap.dedent(f"""\
        --loss=ddpm
        --sampling=ddpm
        --schedule_type=linear
        --sigma_begin=1e-6
        --sigma_end=0.01
        --num_sigmas=50
        --continuous_noise
        --problem=vae
        --ema=False
        --nosnapshot_sampling
        --architecture=TransformerDDPM
        --num_layers=1
        --num_mlp_layers=1
        --data_shape=64,{C}
        --slice_ckpt=
        --batch_size=8
        --learning_rate=1e-3
        --max_steps=4
        --snapshot_freq=2
        --logging_freq=2
        --synthetic
        --synthetic_examples=64
        --model_dir={tmp_path / 'run'}
        """))
    env = dict(os.environ, PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, "-m", "smd_b200.train_ncsn", f"--flagfile={cfg}"], capture_output=True,
                       text=True, timeout=600, env=env, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-3000:]
    r = subprocess.run([sys.executable, "-m", "smd_b200.sample_ncsn", f"--flagfile={cfg}", "--sample_size=16"],
                       capture_output=True, text=True, timeout=600, env=env, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-3000:]
    gen = pickle.load(open(tmp_path / "run" / "samples" / "ncsn" / "generated.pkl", "rb"))
    assert gen.shape == (16, 64, C) and np.isfinite(gen).all()
