"""GPU: a clip pass stores the level-0 correlation volume of each frame pair once, and the backward direction reads it
as its transpose.  Its pyramid and lookup must equal, bit for bit, those of a backward volume built by a GEMM of its
own; the engine's flows must still match the oracle."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import raft as oraft
from prisma_b200._lib import check, fptr, lib
from prisma_b200.seeded_weights import make_raft_weights
from prisma_b200.synthetic import synthetic_frame

pytestmark = pytest.mark.gpu

CH = 256


def _frames(n, h8, w8, seed):
    rng = np.random.default_rng(seed)
    f = rng.standard_normal((n, CH, h8, w8), dtype=np.float32)
    return np.ascontiguousarray(f.astype(np.float16).astype(np.float32))


def _level(h, lvl, b, P, n):
    out = np.full((P, n), np.nan, np.float32)
    check(lib().prisma_flowcorr_read_level(h, lvl, b, 0, P, fptr(out)))
    return out


def _lookup(h, coords):
    B, _, h8, w8 = coords.shape
    out = np.full((B, 324, h8, w8), np.nan, np.float32)
    ms = C.c_float()
    check(lib().prisma_flowcorr_lookup(h, fptr(np.ascontiguousarray(coords)), fptr(out), 1, C.byref(ms)))
    return out


def _border_coords(B, h8, w8, seed):
    """Base grid plus fractional offsets up to 6 px, then on the first rows every combination of x and y at and beyond
    the borders (integer and fractional, negative, on the last row / column, far outside), scaled by 2^l so that it
    lands on the border of level l = 0..3 in turn."""
    rng = np.random.default_rng(seed)
    ys, xs = np.mgrid[0:h8, 0:w8].astype(np.float32)
    c = np.stack([xs, ys])[None] + rng.uniform(-6, 6, (B, 2, h8, w8)).astype(np.float32)
    edge_x = [-1000.0, -8.0, -4.0, -0.25, 0.0, w8 - 1, w8 + 3.75, w8 + 4]
    edge_y = [-1000.0, -8.0, -4.0, -0.25, 0.0, h8 - 1, h8 + 3.75, h8 + 4]
    combos = [(x, y) for y in edge_y for x in edge_x]
    for k, (x, y) in enumerate(combos):
        c[:, 0, k // w8, k % w8] = x * (1 << (k % 4))
        c[:, 1, k // w8, k % w8] = y * (1 << (k % 4))
    return c


@pytest.mark.parametrize("npairs,h8,w8", [(1, 13, 21), (4, 13, 21), (2, 11, 37), (4, 24, 40)])
def test_shared_level0_equals_separate_build(npairs, h8, w8):
    """Pair layout (direction 2p + 1 reads 2p's level 0 transposed) against the default layout with the same frames, where
    every direction has its own level-0 GEMM.  P = 273 and 407 leave a partial last lookup CTA and CTAs that straddle
    image rows; 24 x 40 has neither."""
    P = h8 * w8
    B = 2 * npairs
    fr = _frames(npairs + 1, h8, w8, seed=npairs * 100 + h8)
    f1 = [p + (d & 1) for p in range(npairs) for d in range(2)]
    f2 = [p + 1 - (d & 1) for p in range(npairs) for d in range(2)]
    l = lib()
    shared = C.c_void_p()
    check(l.prisma_flowcorr_create_pairs(0, npairs, h8, w8, C.byref(shared)))
    check(l.prisma_flowcorr_set_frames(shared, fptr(fr)))
    sep = C.c_void_p()
    check(l.prisma_flowcorr_create(0, B, h8, w8, C.byref(sep)))
    check(l.prisma_flowcorr_set_fmaps(sep, fptr(np.ascontiguousarray(fr[f1])), fptr(np.ascontiguousarray(fr[f2]))))
    ms = C.c_float()
    check(l.prisma_flowcorr_build(shared, 1, C.byref(ms)))
    check(l.prisma_flowcorr_build(sep, 1, C.byref(ms)))
    try:
        # the build computes and writes level 0 once per pair
        ws, wp = (C.c_double * 2)(), (C.c_double * 2)()
        check(l.prisma_flowcorr_work(shared, ws))
        check(l.prisma_flowcorr_work(sep, wp))
        assert wp[0] - ws[0] == npairs * 2.0 * P * P * CH
        assert wp[1] - ws[1] == npairs * 4.0 * P * P
        # every level of every direction, all rows: level 0 of a backward direction is the transpose of its partner's
        for lvl in range(4):
            n = (h8 >> lvl) * (w8 >> lvl)
            for b in range(B):
                got, ref = _level(shared, lvl, b, P, n), _level(sep, lvl, b, P, n)
                assert np.array_equal(got, ref), (lvl, b)
                if lvl == 0 and b & 1:
                    assert np.array_equal(got, _level(shared, 0, b - 1, P, n).T)
        # a row window of a shared direction
        part = np.full((5, P), np.nan, np.float32)
        check(l.prisma_flowcorr_read_level(shared, 0, 1, P - 5, 5, fptr(part)))
        assert np.array_equal(part, _level(sep, 0, 1, P, P)[P - 5:])
        # lookups: fractional offsets, borders, far outside
        coords = _border_coords(B, h8, w8, seed=7)
        got, ref = _lookup(shared, coords), _lookup(sep, coords)
        assert not np.isnan(got).any()
        assert np.array_equal(got, ref)
        # the check above compared real samples, not zero padding: about half the level-0 taps of these small maps fall
        # inside the volume (most of the coarse levels' fall outside)
        bwd0 = got[1::2, :81]
        assert np.count_nonzero(bwd0) > 0.4 * bwd0.size
        zero = (np.abs(coords) > 500).any(axis=1)  # far outside: every channel of every level is zero
        assert not got.transpose(0, 2, 3, 1)[zero].any()
        # integer positions (no interpolation): the centre tap of level 0 is the volume entry itself
        ys, xs = np.mgrid[0:h8, 0:w8].astype(np.float32)
        ci = np.ascontiguousarray(np.broadcast_to(np.stack([xs, ys])[None], (B, 2, h8, w8)))
        gi, ri = _lookup(shared, ci), _lookup(sep, ci)
        assert np.array_equal(gi, ri)
        l0 = _level(shared, 0, 1, P, P)
        centre = gi[1, 4 * 9 + 4].reshape(P)
        assert np.array_equal(centre, np.diagonal(l0).astype(np.float16).astype(np.float32))
    finally:
        l.prisma_engine_destroy(shared)
        l.prisma_engine_destroy(sep)


def _oracle_flows(frames_rs, iters):
    sd = make_raft_weights(0)
    imgs = [torch.from_numpy(f).permute(2, 0, 1).float()[None] for f in frames_rs]
    i1 = torch.cat([x for p in range(len(imgs) - 1) for x in (imgs[p], imgs[p + 1])])
    i2 = torch.cat([x for p in range(len(imgs) - 1) for x in (imgs[p + 1], imgs[p])])
    pad = oraft.input_pad(*i1.shape[-2:])
    p1 = torch.nn.functional.pad(i1, pad, mode="replicate")
    p2 = torch.nn.functional.pad(i2, pad, mode="replicate")
    with torch.no_grad():
        _, up = oraft.raft_forward(sd, p1, p2, iters)
    H, W = up.shape[-2:]
    return up[..., pad[2]:H - pad[3], pad[0]:W - pad[1]].permute(0, 2, 3, 1).numpy()


def test_engine_pass_with_shared_level0_matches_oracle():
    """A clip of four pairs with one pair per pass and with four: the flows agree bit for bit, and both directions of
    every pair match the oracle (which builds every direction's volume) to the band's 1e-3 of the largest displacement."""
    from prisma_b200.flow import RaftFlowEngine
    iters = 6
    eng = RaftFlowEngine(make_raft_weights(0), iterations=iters, scale=0.75)
    try:
        frames = np.stack([synthetic_frame(240, 320, t) for t in range(5)])
        outs = {}
        for npp in (1, 4):
            eng.pairs_per_pass = npp
            outs[npp] = eng.infer_clip(frames)
            assert outs[npp]["pairs"] == 4
            assert eng.plan_pairs == npp
        for k in ("fwd", "bwd"):
            assert np.array_equal(outs[1][k], outs[4][k]), k
        hs, ws = eng.out_size(240, 320)
        rs = eng.read_tap("resized", (5, hs, ws, 3)).astype(np.uint8)
        ref = _oracle_flows(list(rs), iters)
        for p in range(4):
            for d, k in enumerate(("fwd", "bwd")):
                r = ref[2 * p + d]
                err = np.abs(outs[4][k][p] - r).max() / np.abs(r).max()
                assert err <= 1e-3, (p, k, err)
    finally:
        eng.close()
