"""H100-native (sm_90a) DDPM noise-prediction hot path (import as ``smd_b200``; see smd_b200/__init__.py)."""
