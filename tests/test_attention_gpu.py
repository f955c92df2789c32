"""GPU: wgmma attention kernel vs torch softmax attention (attention.py:49-62 semantics)."""
import ctypes as C

import numpy as np
import pytest
import torch

from prisma_b200._lib import check, fptr, lib

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("T,heads,scale", [(128, 1, 1.0), (300, 2, 1.0), (2443, 6, 2.0), (1813, 6, 4.0), (77, 3, 1.0)])
def test_attention_matches_torch(T, heads, scale):
    D = heads * 64
    rng = np.random.default_rng(T + heads)
    qkv = (rng.standard_normal((T, 3 * D), dtype=np.float32) * scale).astype(np.float16).astype(np.float32)
    out = np.empty((T, D), np.float32)
    ms = C.c_float()
    check(lib().prisma_debug_attention(0, fptr(qkv), fptr(out), T, heads, 1, C.byref(ms)))
    t = torch.from_numpy(qkv).reshape(T, 3, heads, 64).permute(1, 2, 0, 3)
    q, k, v = t[0] * 0.125, t[1], t[2]
    ref = ((q @ k.transpose(-2, -1)).softmax(-1) @ v).permute(1, 0, 2).reshape(T, D).numpy()
    err = np.abs(out - ref).max()
    # P and the output are rounded to fp16 (rel 2^-11); everything else is fp32
    assert err <= 2e-3 * np.abs(ref).max(), f"max abs err {err} vs max {np.abs(ref).max()}"
