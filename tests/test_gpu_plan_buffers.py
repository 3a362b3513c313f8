"""A training plan and an inference plan run the same forward pass on different buffers.

A training plan keeps every forward activation (one workspace region per layer / block) for the backward pass; an
inference plan overwrites one region per tensor family in place.  Inference on a training plan must still give
bit-identical results, and the training forward's saved activations must be readable by name (smd_debug_buffer) and
match the oracle stage by stage."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import ddpm_oracle as O
from smd_b200 import lib as L
from tests.util import make_inputs, oracle_kwargs, params_torch, rel_l2

pytestmark = pytest.mark.gpu

CASES = {
    # name: (ModelConfig kwargs, arch, batch)
    "heads8_b4": (dict(num_layers=2, num_heads=8, num_mlp_layers=2, channels=42), "TransformerDDPM", 4),   # fused attention
    "heads8_b256": (dict(num_layers=1, num_heads=8, num_mlp_layers=1, channels=42), "TransformerDDPM", 256),  # + fused FFN
    "heads4": (dict(num_layers=2, num_heads=4, num_mlp_layers=1, channels=42), "TransformerDDPM", 3),      # unfused
    "dense": (dict(num_layers=2, channels=512), "DenseDDPM", 8),
}


@pytest.mark.parametrize("case", list(CASES))
def test_training_plan_infers_like_inference_plan(lib, case):
    from smd_b200 import Engine, ModelConfig
    kw, arch, batch = CASES[case]
    cfg = ModelConfig(arch=arch, **kw)
    shape = (32, kw["channels"]) if arch == "TransformerDDPM" else (kw["channels"],)
    engines = [Engine(cfg, max_batch=batch, training=tr) for tr in (True, False)]
    flat = engines[0].init_params(seed=3, perturb=0.02)
    x, t = make_inputs(11, batch, shape)
    rng = np.random.default_rng(5)
    eps = torch.from_numpy(rng.standard_normal((batch, *shape)).astype(np.float32)).cuda()
    used = torch.from_numpy(rng.uniform(0.05, 0.99, (batch,)).astype(np.float32)).cuda()
    xd, td = torch.from_numpy(x).cuda(), torch.from_numpy(t).cuda()
    outs = []
    for eng in engines:
        eng.set_params(flat)
        y = eng.forward(xd, td)
        loss, pred = eng.ddpm_loss(xd, used, eps, want_pred=True)
        torch.cuda.synchronize()
        outs.append((y, loss, pred))
    (y_tr, loss_tr, pred_tr), (y_inf, loss_inf, pred_inf) = outs
    assert torch.equal(y_tr, y_inf)
    assert torch.equal(loss_tr, loss_inf)
    assert torch.equal(pred_tr, pred_inf)


class _DeviceBytes:
    """A workspace region as a uint8 device array, for torch.as_tensor."""

    def __init__(self, ptr: int, nbytes: int):
        self.__cuda_array_interface__ = {"shape": (nbytes,), "typestr": "|u1", "data": (ptr, False), "strides": None,
                                         "version": 3}


def _region(eng, name, shape, dtype):
    ptr, nbytes = C.c_void_p(), C.c_size_t()
    L.check(eng.lib.smd_debug_buffer(eng._plan, name.encode(), C.byref(ptr), C.byref(nbytes)))
    need = int(np.prod(shape)) * torch.tensor([], dtype=dtype).element_size()
    assert need <= nbytes.value, (name, need, nbytes.value)
    raw = torch.as_tensor(_DeviceBytes(ptr.value, nbytes.value), device="cuda")
    return raw[:need].view(dtype).reshape(shape).float().cpu()


def test_saved_activations_match_oracle_trace(lib):
    from smd_b200 import Engine, ModelConfig
    kw = dict(num_layers=2, num_heads=8, num_mlp_layers=2, channels=42)
    batch = 4
    eng = Engine(ModelConfig(**kw), max_batch=batch, training=True)
    flat = eng.init_params(seed=1, perturb=0.02)
    eng.set_params(flat)
    x, t = make_inputs(7, batch, (32, 42))
    xd, td = torch.from_numpy(x).cuda(), torch.from_numpy(t).cuda()
    y = torch.empty_like(xd)
    L.check(eng.lib.smd_debug_forward_save(eng._plan, eng.params.data_ptr(), xd.data_ptr(), td.data_ptr(), batch,
                                           y.data_ptr(), torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    trace = {}
    ref = O.transformer_ddpm(params_torch(eng, flat), torch.from_numpy(x), torch.from_numpy(t), emulate_bf16=True,
                             trace=trace, **oracle_kwargs(eng.cfg))
    assert rel_l2(y, ref) < 1e-2
    M, Md = batch * 32, eng.cfg.mlp_dims
    kinds = {"t.h": ((M, 128), torch.float32), "t.a1_": ((M, 128), torch.bfloat16),
             "t.a2_": ((M, 128), torch.bfloat16), "t.hpre": ((M, Md), torch.bfloat16),
             "t.hid": ((M, Md), torch.bfloat16), "t.a_post": ((M, 128), torch.bfloat16),
             "t.u": ((M, Md), torch.float32), "t.act_out": ((M, Md), torch.bfloat16)}
    ss = _region(eng, "ss", (kw["num_mlp_layers"], batch, 2 * Md), torch.float32)
    checked = 0
    for name, val in trace.items():
        if name.startswith("ss"):
            got = ss[int(name[2:])]
        else:
            shape, dt = kinds[max((k for k in kinds if name.startswith(k)), key=len)]
            got, val = _region(eng, name, shape, dt), val.reshape(shape)
        assert rel_l2(got, val) < 1e-2, name
        checked += 1
    assert checked == 6 * kw["num_layers"] + 2 * kw["num_mlp_layers"] + 4
