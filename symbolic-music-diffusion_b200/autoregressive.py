"""Autoregressive models, same names as the reference's models/autoregressive.py:

  shift_right      models/autoregressive.py:25-33
  TransformerMDN   models/autoregressive.py:36-82 (keywords num_layers, num_heads, num_mlp_layers, mlp_dims,
                   mdn_mixtures); ``model(inputs, shift=True) -> (pi, mu, log_sigma)``

The forward pass is hand-written CUDA behind include/smd.h (smd_mdn_forward).
"""
import numpy as np
import torch

from .nn import ModuleSpec

TransformerMDN = ModuleSpec("TransformerMDN")


def shift_right(x):
    """Shift the input to the right by padding on axis 1 (a zero position in front, the last one dropped)."""
    if isinstance(x, torch.Tensor):
        return torch.cat([torch.zeros_like(x[:, :1]), x[:, :-1]], dim=1)
    x = np.asarray(x)
    pad = [(0, 0)] * x.ndim
    pad[1] = (1, 0)
    return np.pad(x, pad, mode="constant", constant_values=x.dtype.type(0))[:, :-1]
