"""Independent cross-checks of the oracle's building blocks (CPU only).

Upstream ships no golden vectors and cannot run here, so the oracle is "unpinned by the reference".
What CAN be done is to check every primitive it restates against an independent implementation of the same published
algorithm: PyTorch's own LayerNorm / tanh-GELU / SiLU / MultiheadAttention / pre-LN TransformerEncoderLayer / Adam /
clip_grad_norm_, and the closed-form DDPM posterior of Ho et al. 2020 (eqs. 6-7) in float64.  These are different code
bases (ATen kernels, torch.optim) written from the same papers the flax / jax functions implement."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import ddpm_oracle as O

torch.manual_seed(0)


def test_layer_norm_matches_torch_layer_norm():
    x = torch.randn(7, 32, 128, dtype=torch.float64) * 3 + 0.5
    g, b = torch.randn(128, dtype=torch.float64), torch.randn(128, dtype=torch.float64)
    ref = F.layer_norm(x, (128,), g, b, eps=1e-6)          # two-pass variance; flax: E[x^2] - E[x]^2 (same in exact math)
    assert torch.allclose(O.layer_norm(x, g, b), ref, rtol=0, atol=1e-10)
    x32 = x.float()
    assert torch.allclose(O.layer_norm(x32, g.float(), b.float()), ref.float(), rtol=0, atol=5e-5)


def test_activations_match_torch():
    x = torch.linspace(-8, 8, 4001, dtype=torch.float64)
    assert torch.allclose(O.gelu_tanh(x), F.gelu(x, approximate="tanh"), rtol=0, atol=1e-12)
    assert torch.allclose(O.swish(x), F.silu(x), rtol=0, atol=1e-12)


@pytest.mark.parametrize("heads", [4, 8, 16])
def test_self_attention_matches_torch_multihead_attention(heads):
    E, B, S = 128, 3, 32
    p = {"a.qkv.kernel": torch.randn(E, 3 * E, dtype=torch.float64) / math.sqrt(E),
         "a.qkv.bias": torch.randn(3 * E, dtype=torch.float64) * 0.1,
         "a.out.kernel": torch.randn(E, E, dtype=torch.float64) / math.sqrt(E),
         "a.out.bias": torch.randn(E, dtype=torch.float64) * 0.1}
    mha = torch.nn.MultiheadAttention(E, heads, bias=True, batch_first=True, dtype=torch.float64)
    with torch.no_grad():
        mha.in_proj_weight.copy_(p["a.qkv.kernel"].t())        # torch: (3E, E) = [Wq; Wk; Wv], y = x W^T
        mha.in_proj_bias.copy_(p["a.qkv.bias"])
        mha.out_proj.weight.copy_(p["a.out.kernel"].t())
        mha.out_proj.bias.copy_(p["a.out.bias"])
    x = torch.randn(B, S, E, dtype=torch.float64)
    ref, _ = mha(x, x, x, need_weights=False)
    got = O.self_attention(x, p, "a.", heads)
    assert torch.allclose(got, ref, rtol=0, atol=1e-11)


def test_trunk_layer_matches_torch_pre_ln_encoder_layer():
    """One layer of models/ncsn.py:158-168 (LN -> attention -> +x ; LN -> Dense -> gelu -> Dense -> +x) is a pre-LN
    transformer encoder layer: torch.nn.TransformerEncoderLayer(norm_first=True) with the same weights must agree."""
    E, M, H, B, S = 128, 512, 8, 2, 32
    dt = torch.float64
    p = {"in.kernel": torch.eye(E, dtype=dt), "in.bias": torch.zeros(E, dtype=dt)}
    names = {"ln1.scale": (E,), "ln1.bias": (E,), "attn.qkv.kernel": (E, 3 * E), "attn.qkv.bias": (3 * E,),
             "attn.out.kernel": (E, E), "attn.out.bias": (E,), "ln2.scale": (E,), "ln2.bias": (E,),
             "ffn1.kernel": (E, M), "ffn1.bias": (M,), "ffn2.kernel": (M, E), "ffn2.bias": (E,)}
    for n, shp in names.items():
        t = torch.randn(*shp, dtype=dt)
        p["l0." + n] = t / math.sqrt(shp[0]) if len(shp) == 2 else (1 + 0.1 * t if n.endswith("scale") else 0.1 * t)
    layer = torch.nn.TransformerEncoderLayer(E, H, dim_feedforward=M, dropout=0.0, batch_first=True, norm_first=True,
                                             activation=lambda v: F.gelu(v, approximate="tanh"), layer_norm_eps=1e-6,
                                             dtype=dt)
    with torch.no_grad():
        layer.self_attn.in_proj_weight.copy_(p["l0.attn.qkv.kernel"].t()); layer.self_attn.in_proj_bias.copy_(p["l0.attn.qkv.bias"])
        layer.self_attn.out_proj.weight.copy_(p["l0.attn.out.kernel"].t()); layer.self_attn.out_proj.bias.copy_(p["l0.attn.out.bias"])
        layer.norm1.weight.copy_(p["l0.ln1.scale"]); layer.norm1.bias.copy_(p["l0.ln1.bias"])
        layer.norm2.weight.copy_(p["l0.ln2.scale"]); layer.norm2.bias.copy_(p["l0.ln2.bias"])
        layer.linear1.weight.copy_(p["l0.ffn1.kernel"].t()); layer.linear1.bias.copy_(p["l0.ffn1.bias"])
        layer.linear2.weight.copy_(p["l0.ffn2.kernel"].t()); layer.linear2.bias.copy_(p["l0.ffn2.bias"])
    layer.eval()
    x = torch.randn(B, S, E, dtype=dt)
    ref = layer(x)
    # the oracle's layer body, taken from its trace of a 1-layer model (t.h0 = input + positional encoding)
    trace = {}
    full = dict(p)
    for n in ("post_ln.scale", "out_ln.scale"):
        full[n] = torch.ones(E if n.startswith("post") else M, dtype=dt)
    for n in ("post_ln.bias", "out_ln.bias"):
        full[n] = torch.zeros(E if n.startswith("post") else M, dtype=dt)
    full.update({"post.kernel": torch.zeros(E, M, dtype=dt), "post.bias": torch.zeros(M, dtype=dt),
                 "out.kernel": torch.zeros(M, E, dtype=dt), "out.bias": torch.zeros(E, dtype=dt)})
    pe = O.transformer_positional_encoding(S, E, dt)[None]
    O.transformer_ddpm(full, x - pe, torch.ones(B, dtype=dt), num_layers=1, num_heads=H, num_mlp_layers=0, mlp_dims=M,
                       trace=trace)
    assert torch.allclose(trace["t.h0"], x, rtol=0, atol=1e-12)
    assert torch.allclose(trace["t.h2"], ref, rtol=0, atol=1e-10)


def test_adam_matches_torch_optim_adam():
    torch.manual_seed(3)
    p0 = torch.randn(257, dtype=torch.float64)
    w = torch.nn.Parameter(p0.clone())
    opt = torch.optim.Adam([w], lr=1e-3, betas=(0.9, 0.999), eps=1e-8)
    p, m, v = p0.clone(), torch.zeros_like(p0), torch.zeros_like(p0)
    for step in range(25):
        g = torch.randn(257, dtype=torch.float64) * (1.0 + step)
        w.grad = g.clone()
        opt.step()
        p, m, v = O.adam_step(p, g, m, v, step, 1e-3)
        assert torch.allclose(p, w.detach(), rtol=0, atol=1e-12), step


def test_clip_grads_matches_torch_clip_grad_norm():
    torch.manual_seed(4)
    for scale in (0.01, 1.0, 30.0):
        gs = {k: torch.randn(n, dtype=torch.float64) * scale for k, n in (("a", 11), ("b", 333), ("c", 5))}
        ws = [torch.nn.Parameter(torch.zeros_like(g)) for g in gs.values()]
        for w_, g in zip(ws, gs.values()):
            w_.grad = g.clone()
        torch.nn.utils.clip_grad_norm_(ws, 1.0)            # g * min(1, max / (norm + 1e-6))
        got = O.clip_grads(gs, 1.0)                         # g if norm < max else g * (max / norm)
        for w_, g in zip(ws, got.values()):
            assert torch.allclose(g, w_.grad, rtol=2e-6, atol=0)


def test_reverse_coefficients_match_the_ddpm_posterior_in_float64():
    """utils/ebm_utils.py:334-357 against Ho et al. 2020: x0 = (x_t - sqrt(1 - abar) eps) / sqrt(abar);
    q(x_{t-1} | x_t, x0) = N(mu1 x0 + mu2 x_t, sigma^2) with mu1 = sqrt(abar_{t-1}) beta / (1 - abar),
    mu2 = sqrt(alpha) (1 - abar_{t-1}) / (1 - abar), sigma^2 = beta (1 - abar_{t-1}) / (1 - abar)."""
    betas = O.create_noise_schedule(1e-6, 0.01, 1000, "linear").astype(np.float64)
    alphas = 1.0 - betas
    abar = np.cumprod(alphas)
    abar_prev = np.concatenate([[1.0], abar[:-1]])
    c = O.reverse_coefficients(betas.astype(np.float32))
    assert np.allclose(c["sqrt_recip_alpha_prod"], 1.0 / np.sqrt(abar), rtol=2e-6)
    # sqrt(1 / abar - 1) is formed in fp32 like upstream: the subtraction cancels for abar -> 1 (0.7 % at t = 0, pinned
    # as such in tests/test_host_logic.py), so the float64 closed form is compared where abar < 0.99
    far = abar < 0.99
    assert np.allclose(c["sqrt_alpha_prod_m1"][far], np.sqrt(1.0 / abar - 1.0)[far], rtol=1e-4)
    # the same holds for 1 - abar in the posterior coefficients (0.3 % at t = 1 in fp32)
    assert np.allclose(c["mu1"][far], (np.sqrt(abar_prev) * betas / (1.0 - abar))[far], rtol=1e-4)
    assert np.allclose(c["mu2"][far], (np.sqrt(alphas) * (1.0 - abar_prev) / (1.0 - abar))[far], rtol=1e-4)
    assert np.allclose(c["sigma"][far] ** 2, (betas * (1.0 - abar_prev) / (1.0 - abar))[far], rtol=2e-4)
    assert far.sum() > 850


def test_reverse_step_matches_ancestral_sampling_from_the_paper():
    """One reverse step of the oracle (utils/ebm_utils.py:327-397) against Algorithm 2 of Ho et al. with the clipped
    x0-parameterisation, written independently in float64: x0 = clip((x - sqrt(1 - abar) eps) / sqrt(abar), -1, 1),
    x_{t-1} = posterior_mean(x0, x) + sqrt(beta_tilde) z."""
    betas32 = O.create_noise_schedule(1e-6, 0.01, 1000, "linear")
    coef = O.reverse_coefficients(betas32)
    betas = betas32.astype(np.float64)
    alphas = 1.0 - betas
    abar = np.cumprod(alphas)
    abar_prev = np.concatenate([[1.0], abar[:-1]])
    g = torch.Generator().manual_seed(11)
    x = torch.randn(5, 32, 42, generator=g, dtype=torch.float64)
    z = torch.randn(5, 32, 42, generator=g, dtype=torch.float64)
    eps_hat = torch.randn(5, 32, 42, generator=g, dtype=torch.float64) * 0.7
    for t in (999, 700, 400, 150):
        nxt, _, _ = O.reverse_step(lambda s, c: eps_hat, x, t, coef, z)
        x0 = torch.clamp((x - math.sqrt(1.0 - abar[t]) * eps_hat) / math.sqrt(abar[t]), -1.0, 1.0)
        mean = (math.sqrt(abar_prev[t]) * betas[t] / (1.0 - abar[t])) * x0 + \
               (math.sqrt(alphas[t]) * (1.0 - abar_prev[t]) / (1.0 - abar[t])) * x
        ref = mean + math.sqrt(betas[t] * (1.0 - abar_prev[t]) / (1.0 - abar[t])) * z
        assert torch.allclose(nxt, ref, rtol=0, atol=2e-4), t


def test_sinusoidal_encodings_match_the_closed_forms():
    """models/shared.py:33-48 is the timing signal of "Attention is all you need" as tensor2tensor computes it
    (geometric timescales 1 .. 10000 over channels / 2 - 1 steps, [sin | cos]); models/ncsn.py:25-41 is WaveGrad's
    noise-level encoding (same frequencies, argument 5000 * noise).  Written here with pow() instead of exp(log())."""
    S, E = 32, 128
    half = E // 2
    inv_timescale = np.power(10000.0, -np.arange(half, dtype=np.float64) / (half - 1))
    pos = np.arange(S, dtype=np.float64)[:, None] * inv_timescale[None, :]
    ref = np.concatenate([np.sin(pos), np.cos(pos)], axis=1)
    got64 = O.transformer_positional_encoding(S, E, torch.float64).numpy()
    assert np.allclose(got64, ref, rtol=0, atol=1e-12)
    got32 = O.transformer_positional_encoding(S, E, torch.float32).numpy()
    assert np.allclose(got32, ref, rtol=0, atol=2e-5)        # fp32 frequencies times positions up to 31
    noise = np.linspace(0.0026, 1.0, 9)
    arg = (5000.0 * noise)[:, None] * inv_timescale[None, :]
    refn = np.concatenate([np.sin(arg), np.cos(arg)], axis=1)
    gotn = O.noise_encoding(torch.from_numpy(noise), E).numpy()
    assert np.allclose(gotn, refn, rtol=0, atol=1e-9)
