"""The fused epilogue of the shifted-row GEMM (gemm_tc.cuh: GemmEpilogue) feature by feature, through prisma_debug_gemm_ep,
against a float64 model of the same arithmetic.

Most cases use exact GEMMs: A holds small integers and W multiples of 1/64, so every product and partial sum is exact in
fp32 and the accumulator equals the float64 value; what is left to tolerate is the epilogue's own rounding, which the model
carries as an elementwise error bound next to every value.  Cases with random operands add c * 2^-24 * K * (|A| |W|^T) for
the accumulation.  Every destination starts as NaN, with border rows, an extra image and a pitch wider than N: exactly the
mapped (row, column < N) cells must be written.

The reference helpers (row mapper, shifted-row gather, epilogue model) are plain numpy; the tests at the top check them
against torch.nn.functional.conv2d and run without a GPU.
"""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from prisma_b200._lib import DebugEpilogue

U = 2.0 ** -24  # fp32 unit roundoff
ROW_LINEAR, ROW_PADDED, ROW_TOK2PAD, ROW_SHUFFLE, ROW_TOKSKIP, ROW_PAD2TOK = 0, 1, 2, 3, 4, 5
GEOM_KEYS = ("row_map", "img_rows", "in_w", "in_h", "out_wp", "out_img_rows", "sub", "pad", "out_pad", "lead", "out_lead",
             "shuf_s", "shuf_cout")


def _ru(a, b):
    return (a + b - 1) // b * b


# ------------------------------------------------------------------------------------------------ reference model (CPU)
def map_rows(M, row_map=ROW_LINEAR, img_rows=0, in_w=0, in_h=0, out_wp=0, out_img_rows=0, sub=1, pad=1, out_pad=1,
             lead=-1, out_lead=-1, **_):
    """Destination row of every output-space row m < M, or -1 where the row is not stored (all maps but ROW_SHUFFLE)."""
    m = np.arange(M, dtype=np.int64)
    dst, valid = m.copy(), np.ones(M, bool)
    out_ld = out_pad if out_lead < 0 else out_lead
    if row_map in (ROW_PADDED, ROW_PAD2TOK):
        img = m // img_rows if img_rows > 0 else np.zeros_like(m)
        r = m - img * img_rows
        y, x = r // in_w, r % in_w
        ld = pad if lead < 0 else lead
        valid = (y >= ld) & (y < in_h - pad) & (x >= ld) & (x < in_w - pad)
        if row_map == ROW_PAD2TOK:
            ho, wo = -(-(in_h - pad - ld) // sub), -(-(in_w - pad - ld) // sub)
            valid &= ((y - ld) % sub == 0) & ((x - ld) % sub == 0)
            dst = img * (out_img_rows if out_img_rows > 0 else ho * wo) + ((y - ld) // sub) * wo + (x - ld) // sub
        elif sub > 1 or out_wp > 0:
            valid &= ((y - ld) % sub == 0) & ((x - ld) % sub == 0)
            dst = img * out_img_rows + ((y - ld) // sub + out_ld) * out_wp + (x - ld) // sub + out_ld
    elif row_map == ROW_TOKSKIP:
        dst = m + m // in_w + 1
    elif row_map == ROW_TOK2PAD:
        per = in_w * in_h
        img, r = m // per, m % per
        dst = img * out_img_rows + (r // in_w + out_ld) * out_wp + r % in_w + out_ld
    else:
        assert row_map == ROW_LINEAR
    return np.where(valid, dst, -1)


def map_cells(M, N, geom):
    """(dst row, dst column) of every output cell (m < M, n < N); row -1 = not stored.  ROW_SHUFFLE spreads the columns
    n = (dy * s + dx) * cout + co of token (y, x) over the s x s output pixels (y * s + dy, x * s + dx)."""
    n = np.arange(N, dtype=np.int64)
    if geom.get("row_map") != ROW_SHUFFLE:
        return np.repeat(map_rows(M, **geom)[:, None], N, 1), np.broadcast_to(n, (M, N)).copy()
    s, cout = geom["shuf_s"], geom["shuf_cout"]
    out_ld = geom.get("out_pad", 1) if geom.get("out_lead", -1) < 0 else geom["out_lead"]
    m = np.arange(M, dtype=np.int64)
    per = geom["in_w"] * geom["in_h"]
    img, r = m // per, m % per
    ty, tx = r // geom["in_w"], r % geom["in_w"]
    q = n // cout
    rows = (img[:, None] * geom["out_img_rows"] + (ty[:, None] * s + q // s + out_ld) * geom["out_wp"]
            + tx[:, None] * s + q % s + out_ld)
    return rows, np.broadcast_to(n % cout, (M, N)).copy()


def gather_rows(A, offs, M):
    """Shifted-row operand: row m of tap t is A[m + offs[t]], zero outside [0, a_rows)."""
    a_rows, K = A.shape
    out = np.zeros((M, len(offs) * K))
    for t, o in enumerate(offs):
        src = np.arange(M) + o
        ok = (src >= 0) & (src < a_rows)
        out[ok, t * K:(t + 1) * K] = A[src[ok]]
    return out


def ref_acc(A, w, offs, M):
    """D[m, n] = sum_t sum_c A[m + offs[t], c] w[n, t, c] in float64, and sum |A| |w| (the accumulation error scale)."""
    G = gather_rows(A, offs, M)
    wf = w.reshape(w.shape[0], -1)
    return G @ wf.T, np.abs(G) @ np.abs(wf).T


class Geometry:
    """B zero-bordered [Hp][Wp] images stacked image-major: symmetric (`pad` on every side) or shared-border (pad only after
    every row / image, GemmEpilogue::lead == 0); align32 rounds the rows per image up to a multiple of 32 (RAFT maps)."""

    def __init__(self, B, H, W, pad, shared=False, align32=False):
        self.B, self.H, self.W, self.pad, self.shared = B, H, W, pad, shared
        self.Hp, self.Wp = (H + pad, W + pad) if shared else (H + 2 * pad, W + 2 * pad)
        self.img_rows = _ru(self.Hp * self.Wp, 32) if align32 else self.Hp * self.Wp
        self.ld = 0 if shared else pad
        self.rows = B * self.img_rows

    def row(self, b, y, x):
        return b * self.img_rows + (y + self.ld) * self.Wp + x + self.ld

    def pixel_rows(self):  # [B][H][W] row index of every interior pixel
        b, y, x = np.meshgrid(np.arange(self.B), np.arange(self.H), np.arange(self.W), indexing="ij")
        return self.row(b, y, x)

    def embed(self, x_bhwc):
        A = np.zeros((self.rows, x_bhwc.shape[-1]))
        A[self.pixel_rows().ravel()] = x_bhwc.reshape(-1, x_bhwc.shape[-1])
        return A

    def extract(self, D):
        return D[self.pixel_rows()]

    def src_geom(self, sub=1):  # the ROW_PADDED / ROW_PAD2TOK fields describing this map as the GEMM's input space
        return dict(img_rows=self.img_rows, in_w=self.Wp, in_h=self.Hp, pad=self.pad, sub=sub, lead=0 if self.shared else -1)

    def dst_geom(self):  # the destination fields describing this map as a ROW_PADDED / ROW_TOK2PAD destination
        return dict(out_wp=self.Wp, out_img_rows=self.img_rows, out_pad=self.pad, out_lead=0 if self.shared else -1)


def conv_offsets(kh, kw, Wp):
    return [(ky - kh // 2) * Wp + (kx - kw // 2) for ky in range(kh) for kx in range(kw)]


def act_ref(act, x, ex):
    """float64 activation of x, whose absolute error bound is ex -> (value, error bound of the kernel's fp32 result)."""
    if act == 0:
        return x, ex
    if act == 2:
        return np.maximum(x, 0.0), ex
    if act == 1:  # 0.5 x (1 + erff(x / sqrt 2)): erff within 2 ulp, three roundings
        erf = torch.erf(torch.from_numpy(x) / math.sqrt(2.0)).numpy()
        y = 0.5 * x * (1.0 + erf)
        d = 0.5 * (1.0 + erf) + x * np.exp(-0.5 * x * x) / math.sqrt(2.0 * math.pi)
        return y, np.abs(d) * ex + 4 * U * (np.abs(y) + 0.5 * np.abs(x) * (1.0 + np.abs(erf)))
    if act in (3, 6):
        y = 1.0 / (1.0 + np.exp(-x))
        d = y * (1.0 - y)
        # 6: expf + IEEE division (a few ulp); 3: ex2.approx + rcp.approx (~4e-7, plus the rounding of x * log2(e) that
        # __expf's argument takes, relative |x| 2^-24 in the exponential)
        err = 4 * U * y if act == 6 else (4e-7 + np.abs(x) * 2.0 ** -22) * y
        return y, d * ex + err + 1e-36
    if act == 4:  # 1 - 2 / (exp(2x) + 1): ~2e-7 absolute near 0, the exponential's argument rounding elsewhere
        y = np.tanh(x)
        d = 1.0 - y * y
        return y, d * ex + 4e-7 * np.abs(y) + 2.5e-7 + d * np.abs(x) * 2.0 ** -21
    if act == 5:  # nn.Softplus(beta 1, threshold 20): log1pf(expf(x)) below the threshold
        y = np.where(x > 20.0, x, np.log1p(np.exp(np.minimum(x, 20.0))))
        d = 1.0 / (1.0 + np.exp(-x))
        return y, d * ex + 4 * U * np.abs(y) + 1e-36
    raise ValueError(act)


def epilogue_ref(acc, eacc, rows, cols, p):
    """float64 model of epilogue_rows8 (register path) / stage_fragment (TMA path) for the cells (m, n) of acc, stored at
    (rows, cols) (-1 = not stored).  p: host float64 copies of the epilogue's inputs.  Returns value / error-bound arrays."""
    ok = rows >= 0
    r, c = np.where(ok, rows, 0), np.where(ok, cols, 0)

    def at(buf, ld_cols=None):  # an input indexed by destination row (and column)
        return np.where(ok, buf[r, c if ld_cols is None else ld_cols], 0.0)

    N = acc.shape[1]
    n = np.arange(N)
    alpha = p.get("alpha", 1.0)
    bias = p["bias"] if p.get("bias") is not None else np.zeros(N)
    x = alpha * acc + bias
    exact_fma = p.get("bias") is None and math.frexp(alpha)[0] == 0.5  # power-of-two scale, no bias: fmaf is exact
    e = abs(alpha) * eacc + (0.0 if exact_fma else U * np.abs(x))
    if p.get("pre_f32") is not None:
        x = x + at(p["pre_f32"])
        e = e + U * np.abs(x)
    out = {"x": x}
    y, e = act_ref(p.get("act", 0), x, e)
    if p.get("gamma") is not None:
        y = y * p["gamma"]
        e = e * np.abs(p["gamma"]) + U * np.abs(y)
    gru = p.get("gru", 0)
    if gru == 1:  # columns >= 128 (r): r * h -> gru_rh (fp16), nothing else stored
        h = np.where(ok, p["gru_h"][r, np.maximum(c - 128, 0)], 0.0)
        out["rh"], out["erh"] = y * h, e * np.abs(h) + U * np.abs(y * h)
        out["z_cols"] = n < 128
    elif gru == 2:  # h' = (1 - z) h + z q
        z, h = at(p["gru_z"]), at(p["gru_h"])
        yn = (1.0 - z) * h + z * y
        e = np.abs(z) * e + 2 * U * (np.abs(z * y) + np.abs((1.0 - z) * h)) + U * np.abs(h) + U * np.abs(yn)
        y = yn
    for k in ("res_f32", "res_a", "res_b"):
        if p.get(k) is not None:
            y = y + at(p[k])
            e = e + U * np.abs(y)
    out["v"], out["e"] = y, e
    return out


def expected_buffer(shape, rows, cols, vals, tol):
    """NaN-filled float64 image of a destination with vals / tol at the stored cells (rows -1 skipped)."""
    exp, t = np.full(shape, np.nan), np.full(shape, np.nan)
    ok = rows >= 0
    exp[rows[ok], cols[ok]] = vals[ok]
    t[rows[ok], cols[ok]] = tol[ok]
    return exp, t


def assert_cells(got, exp, tol, what):
    """Exactly the expected cells written (the rest still NaN), each within its tolerance."""
    g = got.double().cpu().numpy() if isinstance(got, torch.Tensor) else np.asarray(got, np.float64)
    g = g.reshape(exp.shape)
    want = ~np.isnan(exp)
    wrong = want != ~np.isnan(g)
    assert not wrong.any(), (f"{what}: {int(wrong.sum())} cells written where they must not be or left unwritten, "
                             f"e.g. (row, col) {np.argwhere(wrong)[:4].tolist()}")
    d = np.abs(g - exp)
    bad = want & ~(d <= tol)
    if bad.any():
        i = tuple(int(j) for j in np.argwhere(bad)[0])
        raise AssertionError(f"{what}: {int(bad.sum())} cells out of tolerance; at {i}: got {g[i]!r} want {exp[i]!r} "
                             f"tol {tol[i]:.3g}; max |err| = {float(d[bad].max()):.3g}")


# ------------------------------------------------------------------------------------------------ CPU self-tests
@pytest.mark.parametrize("k,pad,shared,sub,B,H,W", [
    (3, 1, False, 1, 2, 7, 9),
    (5, 2, False, 1, 3, 6, 8),
    (3, 2, False, 1, 2, 5, 7),
    (3, 1, True, 1, 3, 7, 10),
    (5, 2, True, 1, 2, 6, 9),
    (3, 1, False, 2, 2, 9, 11),
    (3, 1, True, 2, 3, 9, 13),
    (5, 2, True, 2, 2, 8, 7),
])
def test_reference_gather_and_padded_map_equal_conv2d(k, pad, shared, sub, B, H, W):
    """The shifted-row gather plus the ROW_PADDED mapping is a 'same' convolution (stride 1, or stride 2 evaluated at stride 1
    and sub-sampled into another geometry) for symmetric and shared-border layouts."""
    rng = np.random.default_rng(k * 100 + pad * 10 + sub + B + H * W)
    Cin, N = 5, 6
    x = rng.standard_normal((B, H, W, Cin))
    w = rng.standard_normal((N, Cin, k, k))
    src = Geometry(B, H, W, pad, shared, align32=shared)
    offs = conv_offsets(k, k, src.Wp)
    acc, _ = ref_acc(src.embed(x), w.transpose(0, 2, 3, 1).reshape(N, k * k, Cin), offs, src.rows)
    geom = dict(row_map=ROW_PADDED, **src.src_geom(sub))
    Ho, Wo = -(-H // sub), -(-W // sub)
    dst = src
    if sub > 1:
        dst = Geometry(B, Ho, Wo, 1, shared, align32=shared)
        geom.update(dst.dst_geom())
    rows = map_rows(src.rows, **geom)
    D = np.full((dst.rows + 7, N), np.nan)
    D[rows[rows >= 0]] = acc[rows >= 0]
    got = dst.extract(D)
    ref = torch.nn.functional.conv2d(torch.from_numpy(x).permute(0, 3, 1, 2), torch.from_numpy(w), stride=sub,
                                     padding=k // 2).permute(0, 2, 3, 1).numpy()
    np.testing.assert_allclose(got, ref, rtol=1e-12, atol=1e-12)
    assert (rows >= 0).sum() == B * Ho * Wo  # every output pixel exactly once
    assert len(np.unique(rows[rows >= 0])) == B * Ho * Wo


def test_reference_pad2tok_and_shuffle_maps():
    """ROW_PAD2TOK lists the interior pixels densely; ROW_SHUFFLE places the s x s sub-pixels of every token (a
    ConvTranspose2d with kernel == stride)."""
    src = Geometry(2, 5, 7, 1, shared=True, align32=True)
    rows = map_rows(src.rows, row_map=ROW_PAD2TOK, **src.src_geom(2), out_img_rows=20)
    b, y, x = np.meshgrid(np.arange(2), np.arange(0, 5, 2), np.arange(0, 7, 2), indexing="ij")
    np.testing.assert_array_equal(rows[src.row(b, y, x)].ravel(), (b * 20 + (y // 2) * 4 + x // 2).ravel())
    assert (rows >= 0).sum() == 2 * 3 * 4
    # shuffle: tokens [B][H][W][cin] -> ConvTranspose2d(k = s = 2)
    rng = np.random.default_rng(5)
    B, H, W, cin, cout, s = 2, 3, 4, 3, 4, 2
    t = rng.standard_normal((B, H, W, cin))
    wt = rng.standard_normal((cin, cout, s, s))
    dst = Geometry(B, H * s, W * s, 1)
    wg = wt.transpose(2, 3, 1, 0).reshape(s * s * cout, cin)  # n = (dy * s + dx) * cout + co
    acc = t.reshape(-1, cin) @ wg.T
    r, c = map_cells(B * H * W, s * s * cout, dict(row_map=ROW_SHUFFLE, in_w=W, in_h=H, shuf_s=s, shuf_cout=cout,
                                                  **dst.dst_geom()))
    D = np.full((dst.rows, cout), np.nan)
    D[r, c] = acc
    ref = torch.nn.functional.conv_transpose2d(torch.from_numpy(t).permute(0, 3, 1, 2), torch.from_numpy(wt), stride=s)
    np.testing.assert_allclose(dst.extract(D), ref.permute(0, 2, 3, 1).numpy(), rtol=1e-12, atol=1e-12)


# ------------------------------------------------------------------------------------------------ GPU plumbing
def _lib():
    from prisma_b200._lib import lib
    return lib()


def _need_gpu():
    assert torch.cuda.is_available(), "the epilogue tests need an H100"


def nan32(rows, cols):
    return torch.full((rows, cols), float("nan"), dtype=torch.float32, device="cuda")


def nan16(rows, cols):
    return torch.full((rows, cols), float("nan"), dtype=torch.float16, device="cuda")


def dev(a, dtype=torch.float32):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dtype).cuda()


def ptr(t):
    return None if t is None else t.data_ptr()


def exact_rows(rng, rows, K, amax=8):
    return rng.integers(-amax, amax + 1, (rows, K)).astype(np.float64)


def exact_w(rng, N, taps, K, wmax=64):
    return rng.integers(-wmax, wmax + 1, (N, taps, K)) / 64.0


def fp16_values(a):
    return a.astype(np.float16).astype(np.float64)


def upload_a16(A, pitch):
    """fp16 [a_rows][pitch]; the columns past a_cols hold NaN (outside the tensor map: they must never be read)."""
    t = torch.full((A.shape[0], pitch), float("nan"), dtype=torch.float16)
    t[:, :A.shape[1]] = torch.from_numpy(A).half()
    return t.cuda()


def upload_w16(w):
    N, taps, K = w.shape
    kc = -(-K // 64)
    t = torch.zeros((_ru(N, 256), taps, kc * 64), dtype=torch.float16)
    t[:N, :, :K] = torch.from_numpy(w).half()
    return t.reshape(_ru(N, 256), -1).cuda()


def _split(v):
    v = np.ascontiguousarray(v, np.float32)
    hi = (v.view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)
    return hi, (v - hi).astype(np.float32)


def upload_a_tf32(A, c_half):
    """[hi | lo] halves of C_half columns each; the columns [C, C_half) of both halves are never read (NaN)."""
    hi, lo = _split(A)
    t = np.full((A.shape[0], 2 * c_half), np.nan, np.float32)
    t[:, :A.shape[1]], t[:, c_half:c_half + A.shape[1]] = hi, lo
    return dev(t)


def upload_w_tf32(w):
    N, taps, K = w.shape
    hi, lo = _split(w)
    t = np.zeros((_ru(N, 256), taps, 3, K), np.float32)
    t[:N, :, 0], t[:N, :, 1], t[:N, :, 2] = hi, hi, lo
    return dev(t.reshape(_ru(N, 256), -1))


def run(A, W, a_cols, M, N, offs, ep, bn=0, tf32=False, c_half=0):
    """One prisma_debug_gemm_ep call; returns its status (negative = refused, message in prisma_last_error)."""
    _need_gpu()
    offs_c = (C.c_int * len(offs))(*offs)
    torch.cuda.synchronize()
    rc = _lib().prisma_debug_gemm_ep(0, A.data_ptr(), A.shape[0], a_cols, A.shape[1], W.data_ptr(), W.shape[0], M, N,
                                     len(offs), offs_c, bn, int(tf32), c_half, C.byref(ep))
    torch.cuda.synchronize()
    return rc


def run_ok(*args, **kw):
    rc = run(*args, **kw)
    assert rc == 0, _lib().prisma_last_error().decode()


def make_ep(**kw):
    """DebugEpilogue from keyword fields; tensors become their device addresses and stay referenced by the struct (a
    tensor freed here would hand its memory to the next allocation while the kernel still reads it)."""
    ep = DebugEpilogue(**{k: (v.data_ptr() if isinstance(v, torch.Tensor) else v) for k, v in kw.items()})
    ep.keep_alive = [v for v in kw.values() if isinstance(v, torch.Tensor)]
    return ep


def host(t):
    return t.double().cpu().numpy()


def check_f16(got, shape, rows, cols, v, e, what):
    exp, tol = expected_buffer(shape, rows, cols, v, e + 2.0 ** -11 * (np.abs(v) + e) + 2.0 ** -25)
    assert_cells(got, exp, tol, what)


# ------------------------------------------------------------------------------------------------ epilogue arithmetic
@pytest.mark.gpu
@pytest.mark.parametrize("act,M,N,K,bn,alpha,pre", [
    (0, 300, 260, 100, 32, 1.0, False),    # no bias: the accumulator itself, bit-exact; N % 32 = 4
    (0, 1000, 88, 72, 128, 0.75, False),   # N % 32 = 24
    (1, 777, 136, 200, 64, 1.0, False),    # exact-erf GELU; N % 32 = 8
    (2, 333, 48, 64, 32, 1.0, False),      # N % 32 = 16
    (3, 520, 200, 136, 256, 1.0, False),   # fast sigmoid
    (3, 300, 264, 96, 128, 1.0, True),     # + pre_f32 before the activation
    (4, 129, 100, 300, 64, 0.5, False),    # fast tanh
    (5, 2000, 120, 200, 128, 1.0, False),  # softplus: crosses the threshold at 20
    (6, 450, 80, 150, 32, 1.0, False),     # sigmoid with expf + IEEE division
    (6, 300, 256, 128, 256, 1.0, False),
])
def test_activation_epilogue_exact_gemm(act, M, N, K, bn, alpha, pre):
    """alpha acc + bias (+ pre_f32) -> activation -> fp32 and fp16 destinations, over pre-activations in about [-150, 150]
    (past the softplus threshold and where __expf / expf overflow inside the sigmoids and tanh)."""
    rng = np.random.default_rng(act * 1000 + M + N + K)
    A = exact_rows(rng, M, K)
    w = exact_w(rng, N, 1, K)
    acc, _ = ref_acc(A, w, [0], M)
    bias = None if act == 0 and alpha == 1.0 else rng.uniform(-8, 8, N).astype(np.float32).astype(np.float64)
    pre_f32 = rng.uniform(-30, 30, (M + 40, N + 12)).astype(np.float32).astype(np.float64) if pre else None
    out32, out16 = nan32(M + 40, N + 12), nan16(M + 40, N + 20)
    ep = make_ep(alpha=alpha, act=act, bias=None if bias is None else dev(bias),
                 pre_f32=None if pre_f32 is None else dev(pre_f32), pre_f32_ld=N + 12,
                 out_f32=out32, out_f32_ld=N + 12, out_f16=out16, out_f16_ld=N + 20)
    run_ok(upload_a16(A, _ru(K, 8) + 8), upload_w16(w), K, M, N, [0], ep, bn=bn)
    rows, cols = map_cells(M, N, {})
    r = epilogue_ref(acc, np.zeros_like(acc), rows, cols, dict(alpha=alpha, bias=bias, act=act, pre_f32=pre_f32))
    if act >= 3:
        assert (r["x"] < -60).any() and (r["x"] > 60).any(), "the pre-activations must cover the overflow ranges"
    exp, tol = expected_buffer(out32.shape, rows, cols, r["v"], r["e"])
    if act == 0 and bias is None:
        assert np.all(tol[~np.isnan(tol)] == 0)
    assert_cells(out32, exp, tol, "out_f32")
    check_f16(out16, out16.shape, rows, cols, r["v"], r["e"], "out_f16")


@pytest.mark.gpu
@pytest.mark.parametrize("path,M,N,K,bn", [
    ("register", 700, 264, 200, 32),
    ("register", 700, 264, 200, 64),
    ("register", 2443, 384, 384, 128),
    ("register", 300, 520, 64, 256),
    ("tma_store", 2443, 384, 384, 128),     # fp32 TMA store: alpha, bias, LayerScale staged in stage_fragment
    ("tma_store", 300, 520, 72, 256),
    ("tma_reduce", 2443, 384, 384, 128),    # x += gamma (alpha acc + b) through the L2 reduce-add
    ("tma_reduce", 300, 264, 200, 256),
    ("tma_reduce", 777, 1024, 128, 256),
    ("register_in_place", 300, 264, 200, 64),
])
def test_layerscale_epilogue(path, M, N, K, bn):
    """LayerScale (gamma) with bias and alpha on every store path; the in-place residual starts from a non-zero x0, so the
    result must be x0 + gamma (alpha acc + b) with gamma applied exactly once."""
    rng = np.random.default_rng(M * 3 + N + K + bn)
    A = exact_rows(rng, M, K)
    w = exact_w(rng, N, 1, K)
    acc, _ = ref_acc(A, w, [0], M)
    bias = rng.uniform(-4, 4, N).astype(np.float32).astype(np.float64)
    gamma = rng.uniform(-2, 2, N).astype(np.float32).astype(np.float64)
    alpha = 0.5
    ld, extra = N + 12, 40
    out = nan32(M + extra, ld)
    in_place = path in ("tma_reduce", "register_in_place")
    x0 = None
    if in_place:
        x0 = np.full((M + extra, ld), np.nan)
        x0[:M, :N] = rng.uniform(-4, 4, (M, N)).astype(np.float32)
        out = dev(x0)
    ep = make_ep(alpha=alpha, bias=dev(bias), gamma=dev(gamma), out_f32=out, out_f32_ld=ld,
                 res_f32=out if in_place else None, res_f32_ld=ld if in_place else 0, tma_store=int(path.startswith("tma")))
    run_ok(upload_a16(A, K), upload_w16(w), K, M, N, [0], ep, bn=bn)
    rows, cols = map_cells(M, N, {})
    r = epilogue_ref(acc, np.zeros_like(acc), rows, cols, dict(alpha=alpha, bias=bias, gamma=gamma, res_f32=x0))
    exp, tol = expected_buffer(out.shape, rows, cols, r["v"], r["e"])
    assert_cells(out, exp, tol, path)


@pytest.mark.gpu
def test_residual_f32_not_in_place_and_tf32_epilogue():
    """res_f32 from another buffer (register path) on the fp16 and the 3xTF32 kernels, with gamma and act 6 / 2."""
    rng = np.random.default_rng(11)
    M, N, K = 900, 200, 96
    A = exact_rows(rng, M, K)
    w = exact_w(rng, N, 1, K)
    acc, _ = ref_acc(A, w, [0], M)
    bias = rng.uniform(-4, 4, N).astype(np.float32).astype(np.float64)
    gamma = rng.uniform(-2, 2, N).astype(np.float32).astype(np.float64)
    res = rng.uniform(-50, 50, (M + 8, N + 4)).astype(np.float32).astype(np.float64)
    rows, cols = map_cells(M, N, {})
    for tf32, act, bn in ((False, 2, 64), (True, 6, 32), (True, 6, 128)):
        out = nan32(M + 8, N + 4)
        ep = make_ep(act=act, bias=dev(bias), gamma=dev(gamma), res_f32=dev(res), res_f32_ld=N + 4, out_f32=out,
                     out_f32_ld=N + 4)
        if tf32:
            run_ok(upload_a_tf32(A, 128), upload_w_tf32(w), K, M, N, [0], ep, bn=bn, tf32=True, c_half=128)
        else:
            run_ok(upload_a16(A, K), upload_w16(w), K, M, N, [0], ep, bn=bn)
        r = epilogue_ref(acc, np.zeros_like(acc), rows, cols, dict(bias=bias, gamma=gamma, act=act, res_f32=res))
        exp, tol = expected_buffer(out.shape, rows, cols, r["v"], r["e"])
        assert_cells(out, exp, tol, f"tf32={tf32} act={act} bn={bn}")


@pytest.mark.gpu
def test_rcu_residual_pair_and_relu_copy():
    """The rcu1_conv2 configuration: 3x3 conv on a padded map (random operands), + bias + res_a + res_b, stored as fp16 x and
    relu(x) copies of the same geometry; border rows and the extra image stay NaN."""
    rng = np.random.default_rng(12)
    g = Geometry(2, 13, 21, 1)
    Cin = N = 64
    x = fp16_values(rng.standard_normal((g.B, g.H, g.W, Cin)))
    A = g.embed(x)
    w = fp16_values(rng.standard_normal((N, 9, Cin)) / 24.0)
    offs = conv_offsets(3, 3, g.Wp)
    acc, mag = ref_acc(A, w, offs, g.rows)
    eacc = U * 9 * Cin * mag
    bias = rng.standard_normal(N).astype(np.float32).astype(np.float64)
    res_a = fp16_values(rng.standard_normal((g.rows, N)))
    res_b = fp16_values(rng.standard_normal((g.rows, N)))
    rows_total = g.rows + g.img_rows
    o16, o16r = nan16(rows_total, N + 8), nan16(rows_total, N + 8)
    ep = make_ep(bias=dev(bias), res_a=dev(res_a, torch.float16), res_a_ld=N, res_b=dev(res_b, torch.float16), res_b_ld=N,
                 out_f16=o16, out_f16_ld=N + 8, out_f16_relu=o16r, out_f16_relu_ld=N + 8, row_map=ROW_PADDED, **g.src_geom())
    run_ok(upload_a16(A, Cin), upload_w16(w), Cin, g.rows, N, offs, ep, bn=64)
    rows, cols = map_cells(g.rows, N, dict(row_map=ROW_PADDED, **g.src_geom()))
    r = epilogue_ref(acc, eacc, rows, cols, dict(bias=bias, res_a=res_a, res_b=res_b))
    check_f16(o16, o16.shape, rows, cols, r["v"], r["e"], "out_f16")
    check_f16(o16r, o16r.shape, rows, cols, np.maximum(r["v"], 0), r["e"], "out_f16_relu")


# ------------------------------------------------------------------------------------------------ row mappings
@pytest.mark.gpu
@pytest.mark.parametrize("k,pad,shared,B,H,W,Cin,N,bn,sub", [
    (3, 1, False, 3, 11, 17, 64, 64, 64, 1),
    (5, 2, False, 3, 9, 14, 32, 40, 32, 1),     # Cin < 64 (TMA box wider than the tensor), N % 32 = 8
    (3, 2, False, 3, 10, 12, 64, 88, 128, 1),   # border 2 around a 3x3 conv, N % 32 = 24
    (3, 1, True, 3, 12, 19, 64, 88, 128, 1),    # shared border (RaftEngine::add_conv): lead = out_lead = 0
    (5, 2, True, 2, 10, 15, 96, 128, 256, 1),
    (3, 1, False, 3, 17, 23, 64, 72, 64, 2),    # stride 2 into another geometry, odd H / W
    (3, 1, True, 2, 19, 25, 64, 96, 128, 2),    # stride 2, shared border on both sides
    (5, 2, False, 2, 13, 11, 48, 36, 32, 2),
])
def test_row_padded_conv(k, pad, shared, B, H, W, Cin, N, bn, sub):
    """ROW_PADDED convolutions: only interior pixels (every sub-th one) are stored, at their place in the destination
    geometry; borders, alignment rows and the extra image stay NaN."""
    rng = np.random.default_rng(k + pad * 7 + B * 31 + H * W + sub)
    src = Geometry(B, H, W, pad, shared, align32=shared)
    A = src.embed(exact_rows(rng, B * H * W, Cin).reshape(B, H, W, Cin))
    w = exact_w(rng, N, k * k, Cin, wmax=16)
    offs = conv_offsets(k, k, src.Wp)
    acc, _ = ref_acc(A, w, offs, src.rows)
    bias = rng.uniform(-2, 2, N).astype(np.float32).astype(np.float64)
    geom = dict(row_map=ROW_PADDED, **src.src_geom(sub))
    dst = src
    if sub > 1:
        dst = Geometry(B, -(-H // sub), -(-W // sub), 1, shared, align32=shared)
        geom.update(dst.dst_geom())
    rows_total = dst.rows + dst.img_rows
    out32, out16 = nan32(rows_total, N + 4), nan16(rows_total, N + 12)
    ep = make_ep(bias=dev(bias), act=2, out_f32=out32, out_f32_ld=N + 4, out_f16=out16, out_f16_ld=N + 12, **geom)
    run_ok(upload_a16(A, _ru(Cin, 8)), upload_w16(w), Cin, src.rows, N, offs, ep, bn=bn)
    rows, cols = map_cells(src.rows, N, geom)
    assert (rows[:, 0] >= 0).sum() == B * -(-H // sub) * -(-W // sub)
    r = epilogue_ref(acc, np.zeros_like(acc), rows, cols, dict(bias=bias, act=2))
    exp, tol = expected_buffer(out32.shape, rows, cols, r["v"], r["e"])
    assert_cells(out32, exp, tol, "out_f32")
    check_f16(out16, out16.shape, rows, cols, r["v"], r["e"], "out_f16")


def _dense_map_case(kind, rng):
    """(A rows, a_cols, w, offs, M, N, bn, geom, destination rows) of one row-map case."""
    if kind in ("pad2tok_s1", "pad2tok_s2"):
        sub = 1 if kind == "pad2tok_s1" else 2
        src = Geometry(2, 15, 21, 1) if sub == 1 else Geometry(2, 17, 23, 1, shared=True, align32=True)
        Ho, Wo = -(-src.H // sub), -(-src.W // sub)
        per = Ho * Wo + (13 if sub == 1 else 5)  # out_img_rows: a gap after every image that must stay NaN
        A = src.embed(exact_rows(rng, src.B * src.H * src.W, 64).reshape(src.B, src.H, src.W, 64))
        geom = dict(row_map=ROW_PAD2TOK, out_img_rows=per, **src.src_geom(sub))
        return A, 64, exact_w(rng, 100, 9, 64, wmax=16), conv_offsets(3, 3, src.Wp), src.rows, 100, 64, geom, src.B * per + 50
    if kind in ("tok2pad", "tok2pad_lead0"):
        B, H, W = 2, 13, 18
        dst = Geometry(B, H, W, 1) if kind == "tok2pad" else Geometry(B, H, W, 2, shared=True, align32=True)
        geom = dict(row_map=ROW_TOK2PAD, in_w=W, in_h=H, **dst.dst_geom())
        if kind == "tok2pad":
            geom["out_img_rows"] = dst.img_rows + 7
        M = B * H * W
        return (exact_rows(rng, M, 192), 192, exact_w(rng, 64, 1, 192), [0], M, 64, 64, geom,
                B * geom["out_img_rows"] + 40)
    if kind == "tokskip":
        B, P = 3, 37
        M = B * P
        return exact_rows(rng, M, 200), 200, exact_w(rng, 100, 1, 200), [0], M, 100, 32, dict(row_map=ROW_TOKSKIP, in_w=P), \
            B * (P + 1) + 9
    if kind in ("shuffle2", "shuffle4"):
        B, H, W, s, cout = (2, 7, 9, 2, 36) if kind == "shuffle2" else (2, 5, 6, 4, 16)
        dst = Geometry(B, H * s, W * s, 1)
        geom = dict(row_map=ROW_SHUFFLE, in_w=W, in_h=H, shuf_s=s, shuf_cout=cout, **dst.dst_geom())
        M, N = B * H * W, s * s * cout
        return exact_rows(rng, M, 96), 96, exact_w(rng, N, 1, 96), [0], M, N, 64 if s == 2 else 128, geom, \
            dst.rows + dst.img_rows
    raise ValueError(kind)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["pad2tok_s1", "pad2tok_s2", "tok2pad", "tok2pad_lead0", "tokskip", "shuffle2", "shuffle4"])
def test_row_maps(kind):
    """ROW_PAD2TOK (sub 1 / 2, out_img_rows), ROW_TOK2PAD (symmetric and shared-border destination), ROW_TOKSKIP (the cls
    rows stay untouched; res_f32 is read by destination row like the patch embed's pos-embed) and ROW_SHUFFLE (s 2 / 4)."""
    rng = np.random.default_rng(sum(map(ord, kind)))
    A, a_cols, w, offs, M, N, bn, geom, dst_rows = _dense_map_case(kind, rng)
    acc, _ = ref_acc(A, w, offs, M)
    bias = rng.uniform(-2, 2, N).astype(np.float32).astype(np.float64)
    cout = geom.get("shuf_cout") or N
    res = rng.uniform(-8, 8, (dst_rows, cout + 4)).astype(np.float32).astype(np.float64)
    out32, out16 = nan32(dst_rows, cout + 4), nan16(dst_rows, cout + 8)
    ep = make_ep(bias=dev(bias), act=2, res_f32=dev(res), res_f32_ld=cout + 4, out_f32=out32, out_f32_ld=cout + 4,
                 out_f16=out16, out_f16_ld=cout + 8, **geom)
    run_ok(upload_a16(A, _ru(a_cols, 8)), upload_w16(w), a_cols, M, N, offs, ep, bn=bn)
    rows, cols = map_cells(M, N, geom)
    r = epilogue_ref(acc, np.zeros_like(acc), rows, cols, dict(bias=bias, act=2, res_f32=res))
    exp, tol = expected_buffer(out32.shape, rows, cols, r["v"], r["e"])
    assert_cells(out32, exp, tol, "out_f32")
    check_f16(out16, out16.shape, rows, cols, r["v"], r["e"], "out_f16")


# ------------------------------------------------------------------------------------------------ fused head, statistics, GRU
@pytest.mark.gpu
@pytest.mark.parametrize("bn,copy", [(32, False), (32, True), (64, True)])
def test_dpt_head(bn, copy):
    """output_conv2_fused: depth = relu(head_b + sum_j head_w[j] relu(acc[j] + bias[j])) written dense [B][H][W], and
    optionally the 32 ReLU'd activations as fp16 rows of the same dense index."""
    rng = np.random.default_rng(40 + bn + copy)
    g = Geometry(2, 14, 19, 1)
    Cin, N = 64, 32
    A = g.embed(exact_rows(rng, g.B * g.H * g.W, Cin).reshape(g.B, g.H, g.W, Cin))
    w = exact_w(rng, N, 9, Cin, wmax=8)
    offs = conv_offsets(3, 3, g.Wp)
    acc, _ = ref_acc(A, w, offs, g.rows)
    bias = rng.uniform(-4, 4, N).astype(np.float32).astype(np.float64)
    hw = rng.uniform(-1, 1, N).astype(np.float32).astype(np.float64)
    hb = float(np.float32(0.375))
    npix = g.B * g.H * g.W
    head = nan32(npix + 50, 1)
    act32 = nan16(npix + 50, 40) if copy else None
    ep = make_ep(bias=dev(bias), act=2, head_w=dev(hw), head_b=hb, head_out=head, out_f16=act32, out_f16_ld=40 if copy else 0,
                 row_map=ROW_PADDED, **g.src_geom())
    run_ok(upload_a16(A, Cin), upload_w16(w), Cin, g.rows, N, offs, ep, bn=bn)
    pix_rows = g.pixel_rows().ravel()
    hv = np.maximum(acc[pix_rows] + bias, 0.0)  # [npix][32]
    ehv = U * np.abs(acc[pix_rows] + bias)
    depth = hb + hv @ hw
    edepth = ehv @ np.abs(hw) + 34 * U * (abs(hb) + np.abs(hv) @ np.abs(hw))
    pix = np.arange(npix)
    exp, tol = expected_buffer(head.shape, pix, np.zeros_like(pix), np.maximum(depth, 0), edepth)
    assert_cells(head, exp, tol, "head_out")
    if copy:
        prow, pcol = np.repeat(pix[:, None], N, 1), np.broadcast_to(np.arange(N), (npix, N))
        check_f16(act32, act32.shape, prow, pcol, hv, ehv, "head out_f16")


@pytest.mark.gpu
@pytest.mark.parametrize("sub,N,bn", [(1, 64, 64), (2, 64, 32), (1, 96, 128), (2, 128, 256)])
def test_instnorm_slab_statistics(sub, N, bn):
    """stat_part of a ROW_PAD2TOK conv in the RAFT layout (shared border, images of a multiple of 32 rows, B = 2): every
    32-row slab of every computed tile writes the sum and sum of squares of its valid stored values (random operands);
    slabs without a valid row hold exact zeros; nothing past round_up(M, 128) / 32 slabs is written."""
    rng = np.random.default_rng(60 + sub + N + bn)
    src = Geometry(2, 11, 29, 1, shared=True, align32=True)
    Cin = 64
    A = src.embed(fp16_values(rng.standard_normal((src.B, src.H, src.W, Cin))))
    w = fp16_values(rng.standard_normal((N, 9, Cin)) / 24.0)
    offs = conv_offsets(3, 3, src.Wp)
    M = src.rows
    acc, mag = ref_acc(A, w, offs, M)
    eacc = U * 9 * Cin * mag
    bias = rng.standard_normal(N).astype(np.float32).astype(np.float64)
    Ho, Wo = -(-src.H // sub), -(-src.W // sub)
    nslab = _ru(M, 128) // 32
    dense = nan32(src.B * Ho * Wo + 20, N)
    stats = nan32((nslab + 6) * 2, N)
    geom = dict(row_map=ROW_PAD2TOK, **src.src_geom(sub))
    ep = make_ep(bias=dev(bias), out_f32=dense, out_f32_ld=N, stat_part=stats, **geom)
    run_ok(upload_a16(A, Cin), upload_w16(w), Cin, M, N, offs, ep, bn=bn)
    rows, cols = map_cells(M, N, geom)
    r = epilogue_ref(acc, eacc, rows, cols, dict(bias=bias))
    exp, tol = expected_buffer(dense.shape, rows, cols, r["v"], r["e"])
    assert_cells(dense, exp, tol, "dense out_f32")
    ok = np.zeros((nslab * 32, N), bool)
    ok[:M] = rows >= 0
    v = np.zeros((nslab * 32, N))
    e = np.zeros((nslab * 32, N))
    v[:M], e[:M] = np.where(rows >= 0, r["v"], 0), np.where(rows >= 0, r["e"], 0)
    v, e = v.reshape(nslab, 32, N), e.reshape(nslab, 32, N)
    s1, s2 = v.sum(1), (v * v).sum(1)
    t1 = e.sum(1) + 32 * U * np.abs(v).sum(1)
    t2 = (2 * np.abs(v) * e + e * e).sum(1) + 34 * U * (v * v).sum(1)
    exp = np.full((nslab + 6, 2, N), np.nan)
    tol = np.full((nslab + 6, 2, N), np.nan)
    exp[:nslab, 0], exp[:nslab, 1], tol[:nslab, 0], tol[:nslab, 1] = s1, s2, t1, t2
    empty = ~ok.reshape(nslab, 32, N).any(1)
    assert empty.any() and (~empty).any()
    tol[:nslab][np.repeat(empty[:, None, :], 2, 1)] = 0.0  # slabs without a valid row: exact zeros
    assert_cells(stats, exp.reshape(-1, N), tol.reshape(-1, N), "stat_part")


@pytest.mark.gpu
@pytest.mark.parametrize("gru,bn", [(1, 128), (1, 256), (2, 64), (2, 128)])
def test_convgru_epilogue(gru, bn):
    """The ConvGRU gate epilogues in the RaftEngine::add_conv layout (1x5 / 5x1 taps, shared border 2, B = 2):
    gru 1 (N = 256, sigmoid): z -> out_f32 columns [0, 128) only, r * h -> gru_rh (fp16);
    gru 2 (N = 128, tanh): h' = (1 - z) h + z q in place of h (fp32) plus the fp16 operand copy.
    gru_h has pitch 128, gru_z pitch 256 (its columns >= 128 are NaN: never read), both indexed by destination row."""
    rng = np.random.default_rng(80 + gru * 10 + bn)
    src = Geometry(2, 9, 22, 2, shared=True, align32=True)
    Cin = 96
    A = src.embed(exact_rows(rng, src.B * src.H * src.W, Cin).reshape(src.B, src.H, src.W, Cin))
    kh, kw = (1, 5) if gru == 1 else (5, 1)
    N = 256 if gru == 1 else 128
    w = exact_w(rng, N, kh * kw, Cin, wmax=8)
    offs = conv_offsets(kh, kw, src.Wp)
    M = src.rows
    acc, _ = ref_acc(A, w, offs, M)
    bias = rng.uniform(-2, 2, N).astype(np.float32).astype(np.float64)
    geom = dict(row_map=ROW_PADDED, **src.src_geom())
    rows, cols = map_cells(M, N, geom)
    h0 = rng.uniform(-1, 1, (M, 128)).astype(np.float32).astype(np.float64)
    A_dev, W_dev = upload_a16(A, 104), upload_w16(w)
    if gru == 1:
        out, rh = nan32(M + 64, 264), nan16(M + 64, 136)
        ep = make_ep(bias=dev(bias), act=3, out_f32=out, out_f32_ld=264, gru=1, gru_h=dev(h0), gru_rh=rh, gru_rh_ld=136, **geom)
        run_ok(A_dev, W_dev, Cin, M, N, offs, ep, bn=bn)
        r = epilogue_ref(acc, np.zeros_like(acc), rows, cols, dict(bias=bias, act=3, gru=1, gru_h=h0))
        zc = r["z_cols"]
        exp, tol = expected_buffer(out.shape, rows[:, zc], cols[:, zc], r["v"][:, zc], r["e"][:, zc])
        assert_cells(out, exp, tol, "z (out_f32)")
        check_f16(rh, rh.shape, rows[:, ~zc], cols[:, ~zc] - 128, r["rh"][:, ~zc], r["erh"][:, ~zc], "r * h (gru_rh)")
    else:
        z = np.full((M, 256), np.nan)
        z[:, :128] = rng.uniform(0, 1, (M, 128)).astype(np.float32)
        h = dev(h0)
        out16 = nan16(M + 64, 136)
        ep = make_ep(bias=dev(bias), act=4, out_f32=h, out_f32_ld=128, out_f16=out16, out_f16_ld=136, gru=2, gru_h=h,
                     gru_z=dev(z), **geom)
        run_ok(A_dev, W_dev, Cin, M, N, offs, ep, bn=bn)
        r = epilogue_ref(acc, np.zeros_like(acc), rows, cols, dict(bias=bias, act=4, gru=2, gru_h=h0, gru_z=z))
        stored = rows >= 0
        exp = np.where(stored, r["v"], h0)  # rows that are not stored keep h
        tol = np.where(stored, r["e"], 0.0)
        assert_cells(h, exp, tol, "h' (out_f32, in place)")
        check_f16(out16, out16.shape, rows, cols, r["v"], r["e"], "h' (out_f16)")


# ------------------------------------------------------------------------------------------------ m_dev, 3xTF32
@pytest.mark.gpu
@pytest.mark.parametrize("tf32", [False, True])
def test_device_row_count(tf32):
    """m_dev: only the first round_up(*m_dev, 128) rows (at most M) are computed and stored -- the SOLOv2 mask GEMMs
    (fp16 with the fast sigmoid, 3xTF32 with the IEEE one)."""
    rng = np.random.default_rng(90 + tf32)
    M, N, K = 500, 200, 64
    A = exact_rows(rng, M, K)
    w = exact_w(rng, N, 1, K)
    acc, _ = ref_acc(A, w, [0], M)
    bias = rng.uniform(-4, 4, N).astype(np.float32).astype(np.float64)
    act = 6 if tf32 else 3
    A_dev = upload_a_tf32(A, 96) if tf32 else upload_a16(A, K)
    W_dev = upload_w_tf32(w) if tf32 else upload_w16(w)
    rows_all, cols = map_cells(M, N, {})
    r = epilogue_ref(acc, np.zeros_like(acc), rows_all, cols, dict(bias=bias, act=act))
    for m in (0, 1, 127, 128, 129, M, M + 50):
        m_dev = torch.tensor([m], dtype=torch.int32, device="cuda")
        shape = (M + 20, N + 12)
        out = nan32(*shape) if tf32 else nan16(*shape)
        ep = make_ep(bias=dev(bias), act=act, m_dev=m_dev, **({"out_f32": out, "out_f32_ld": N + 12} if tf32 else
                                                               {"out_f16": out, "out_f16_ld": N + 12}))
        run_ok(A_dev, W_dev, K, M, N, [0], ep, tf32=tf32, c_half=96 if tf32 else 0)
        rows = np.where(rows_all < min(M, _ru(m, 128)), rows_all, -1)
        if tf32:
            exp, tol = expected_buffer(shape, rows, cols, r["v"], r["e"])
            assert_cells(out, exp, tol, f"m_dev={m}")
        else:
            check_f16(out, shape, rows, cols, r["v"], r["e"], f"m_dev={m}")


@pytest.mark.gpu
def test_tf32x3_pad2tok_stride2_sigmoid():
    """The SOLOv2 fp32-class head conv: 3xTF32, 3x3 taps over a padded fp32 [hi | lo] map using C of its C_half channels,
    ROW_PAD2TOK with sub 2, act 6, out_f32; random fp32 operands under the fp32-class bound of test_gemm_tf32x3_is_fp32_class
    (6e-7 of sum |a| |w|) carried through the sigmoid."""
    rng = np.random.default_rng(95)
    src = Geometry(2, 19, 27, 1)
    Cin, c_half, N = 64, 96, 72
    x = (rng.standard_normal((src.B, src.H, src.W, Cin)) * rng.uniform(0.1, 10, (src.B, src.H, src.W, 1))).astype(np.float32)
    A = src.embed(x.astype(np.float64))
    w = (rng.standard_normal((N, 9, Cin)) / 24.0).astype(np.float32).astype(np.float64)
    offs = conv_offsets(3, 3, src.Wp)
    acc, mag = ref_acc(A, w, offs, src.rows)
    bias = rng.standard_normal(N).astype(np.float32).astype(np.float64)
    Ho, Wo = -(-src.H // 2), -(-src.W // 2)
    geom = dict(row_map=ROW_PAD2TOK, **src.src_geom(2))
    out = nan32(src.B * Ho * Wo + 30, N + 8)
    ep = make_ep(bias=dev(bias), act=6, out_f32=out, out_f32_ld=N + 8, **geom)
    run_ok(upload_a_tf32(A, c_half), upload_w_tf32(w), Cin, src.rows, N, offs, ep, tf32=True, c_half=c_half)
    rows, cols = map_cells(src.rows, N, geom)
    r = epilogue_ref(acc, 6e-7 * (mag + np.abs(bias)), rows, cols, dict(bias=bias, act=6))
    exp, tol = expected_buffer(out.shape, rows, cols, r["v"], r["e"])
    assert_cells(out, exp, tol, "3xTF32 out_f32")


# ------------------------------------------------------------------------------------------------ refused configurations
REFUSED = {
    "tma_store with a row map": dict(tma_store=1, row_map=ROW_TOKSKIP, in_w=64),
    "tma_store with a residual not in place": dict(tma_store=1, res_f32="other"),
    "tma_store with an activation on fp32": dict(tma_store=1, act=3),
    "tma_store with stat_part": dict(tma_store=1, stat_part="stats"),
    "tma_store with pre_f32": dict(tma_store=1, pre_f32="other"),
    "tma_store with a relu copy": dict(tma_store=1, out_f16_relu="half"),
    "tma_store with fp32 and fp16 outputs": dict(tma_store=1, out_f16="half"),
    "tma_store fp16 with LayerScale": dict(tma_store=1, out_f32=None, out_f16="half", gamma="vec"),
    "shuffle with shuf_cout % 4 != 0": dict(row_map=ROW_SHUFFLE, in_w=8, in_h=8, shuf_s=2, shuf_cout=30, out_wp=18,
                                            out_img_rows=324, N=120),
    "shuffle with N != s^2 cout": dict(row_map=ROW_SHUFFLE, in_w=8, in_h=8, shuf_s=2, shuf_cout=32, out_wp=18,
                                       out_img_rows=324, N=96),
    "head with N != 32": dict(head_w="vec", head_out="other", bias="vec", row_map=ROW_PADDED, in_w=16, in_h=16, N=64),
    "head without a bias": dict(head_w="vec", head_out="other", row_map=ROW_PADDED, in_w=16, in_h=16, N=32),
    "gru 1 with N != 256": dict(gru=1, gru_h="other", gru_rh="half", N=128),
    "gru 2 with N != 128": dict(gru=2, gru_h="other", gru_z="other", N=256),
    "gru on the 3xTF32 path": dict(gru=2, gru_h="other", gru_z="other", N=128, tf32=True),
    "tma_store on the 3xTF32 path": dict(tma_store=1, tf32=True),
    "force_bn 256 on the 3xTF32 path": dict(tf32=True, bn=256),
    "force_bn 512": dict(bn=512),
}


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(REFUSED))
def test_refused_configurations(case):
    """Combinations the epilogue cannot store correctly are refused by gemm_prepare with a message; nothing is launched
    (the destination stays NaN)."""
    cfg = dict(REFUSED[case])
    N = cfg.pop("N", 128)
    tf32 = cfg.pop("tf32", False)
    bn = cfg.pop("bn", 128)
    M, K = 256, 64
    rng = np.random.default_rng(7)
    A = exact_rows(rng, M, K)
    w = exact_w(rng, 256, 1, K)
    out = nan32(M, 256)
    bufs = {"other": dev(np.zeros((M, 256))), "stats": nan32(64, 256), "half": nan16(M, 256), "vec": dev(np.ones(256))}
    fields = dict(out_f32=out, out_f32_ld=256)
    for k, v in cfg.items():
        fields[k] = bufs[v] if isinstance(v, str) else v
        if k in ("res_f32", "pre_f32", "out_f16", "out_f16_relu"):
            fields[k + "_ld"] = 256
    ep = make_ep(**fields)
    if tf32:
        rc = run(upload_a_tf32(A, K), upload_w_tf32(w), K, M, N, [0], ep, bn=bn, tf32=True, c_half=K)
    else:
        rc = run(upload_a16(A, K), upload_w16(w), K, M, N, [0], ep, bn=bn)
    assert rc < 0, f"{case}: accepted"
    assert "gemm" in _lib().prisma_last_error().decode()
    assert torch.isnan(out).all() and torch.isnan(bufs["half"].float()).all() and torch.isnan(bufs["stats"]).all()


@pytest.mark.gpu
def test_epilogue_struct_size_is_checked():
    _need_gpu()
    ep = make_ep(size=C.sizeof(DebugEpilogue) - 8)
    A, W = torch.zeros((128, 64), dtype=torch.float16, device="cuda"), torch.zeros((256, 64), dtype=torch.float16, device="cuda")
    assert run(A, W, 64, 128, 128, [0], ep) < 0
    assert "size" in _lib().prisma_last_error().decode()
