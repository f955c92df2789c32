"""Host-side mirror of the reference Depth-Anything band interface on top of the C ABI.

Mirrors bands/depth_anything.py: `init_model()` (:48-76) -> `DepthAnythingEngine(...)`,
`infer(img, normalize=False)` (:100-143) -> `engine.infer(img)`, and the per-frame video encode
(:215-221) -> `engine.infer_encoded(img)`.  All arithmetic happens in libprisma_b200.so.
"""
import ctypes as C

import numpy as np

from ._lib import PrismaError, check, fptr, lib, u8ptr, c_i64_p, c_u8_p

# save_point_cloud's vertex dtype (bands/common/geom.py:31-32): 15-byte packed little-endian records
PLY_VERTEX_DTYPE = np.dtype([("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("red", "u1"), ("green", "u1"), ("blue", "u1")])


def da_net_size(width, height):
    """Resize.get_size with the band's settings (d_anything/util/transform.py:111-166), host logic only."""
    sh, sw = 518.0 / height, 518.0 / width
    if sw > sh:
        sh = sw
    else:
        sw = sh

    def constrain(x):
        y = int(np.round(x / 14) * 14)
        if y < 518:
            y = int(np.ceil(x / 14) * 14)
        return y

    return constrain(sw * width), constrain(sh * height)


class _Pinned:
    def __init__(self, nbytes):
        self.ptr = C.c_void_p()
        check(lib().prisma_host_alloc(nbytes, C.byref(self.ptr)))

    def __del__(self):
        try:
            lib().prisma_host_free(self.ptr)
        except Exception:
            pass


def pinned_empty(shape, dtype):
    """numpy array over page-locked host memory (prisma_host_alloc); freed when the array and its views are gone."""
    dtype = np.dtype(dtype)
    nbytes = int(np.prod(shape)) * dtype.itemsize
    owner = _Pinned(max(nbytes, 1))
    buf = (C.c_uint8 * nbytes).from_address(owner.ptr.value)
    buf._owner = owner
    return np.frombuffer(buf, dtype=dtype).reshape(shape)


class DepthAnythingEngine:
    """One engine per (GPU, band).  Not re-entrant; owns device memory, stream and weights."""

    def __init__(self, encoder="vitl", state_dict=None, device=0):
        self._h = C.c_void_p()
        self.encoder = encoder
        self.device = device
        check(lib().prisma_depth_create(encoder.encode(), device, C.byref(self._h)))
        if state_dict is not None:
            self.load_state_dict(state_dict)

    def load_state_dict(self, state_dict):
        """Weight converter: accepts the reference DPT_DINOv2 state_dict (torch tensors or numpy arrays)."""
        l = lib()
        for name, t in state_dict.items():
            a = t.detach().cpu().numpy() if hasattr(t, "detach") else np.asarray(t)
            if a.dtype.kind != "f":
                continue  # e.g. num_batches_tracked
            a = np.ascontiguousarray(a, dtype=np.float32)
            shape = (C.c_int64 * max(a.ndim, 1))(*(a.shape if a.ndim else (1,)))
            check(l.prisma_depth_load_tensor(self._h, name.encode(), fptr(a), C.cast(shape, c_i64_p), max(a.ndim, 1)))
        check(l.prisma_depth_finalize(self._h))

    def infer(self, img, normalize=False):
        """HxWx3 u8 RGB -> HxW f32 depth == bands/depth_anything.py:infer(img, normalize) (--metric none)."""
        pred, _, _, _ = self._run(img, want_depth=True, want_rgb=False)
        if normalize:
            dmin, dmax = pred.min(), pred.max()
            if dmax - dmin > np.finfo("float").eps:
                pred = (pred - dmin) / (dmax - dmin)
        return pred

    def infer_encoded(self, img, want_depth=False):
        """One video frame: (rgb u8 HxWx3, min, max[, depth]) == process_video's loop body (:206-221)."""
        pred, rgb, dmin, dmax = self._run(img, want_depth=want_depth, want_rgb=True)
        return (rgb, dmin, dmax, pred) if want_depth else (rgb, dmin, dmax)

    def _run(self, img, want_depth, want_rgb):
        img = np.ascontiguousarray(img)
        if img.dtype != np.uint8 or img.ndim != 3 or img.shape[2] != 3:
            raise PrismaError("expected an HxWx3 uint8 RGB frame")
        h, w = img.shape[:2]
        pred = np.empty((h, w), np.float32) if want_depth else None
        rgb = np.empty((h, w, 3), np.uint8) if want_rgb else None
        dmin, dmax = C.c_float(), C.c_float()
        check(lib().prisma_depth_infer(self._h, u8ptr(img), h, w, fptr(pred),
                                       u8ptr(rgb), C.byref(dmin), C.byref(dmax)))
        return pred, rgb, dmin.value, dmax.value

    def infer_batch(self, frames, want_depth=False, want_rgb=True):
        """n frames of one size in one pass: (rgb [n,H,W,3] u8 | None, mins [n], maxs [n], depth [n,H,W] f32 | None).
        Identical results to n infer_encoded() calls; the video loop of the band uses this to fill the GPU."""
        x = np.ascontiguousarray(np.stack(frames) if not isinstance(frames, np.ndarray) else frames)
        if x.dtype != np.uint8 or x.ndim != 4 or x.shape[3] != 3:
            raise PrismaError("expected n HxWx3 uint8 RGB frames")
        n, h, w = x.shape[:3]
        pred = np.empty((n, h, w), np.float32) if want_depth else None
        rgb = np.empty((n, h, w, 3), np.uint8) if want_rgb else None
        mins = np.empty(n, np.float32)
        maxs = np.empty(n, np.float32)
        check(lib().prisma_depth_infer_batch(self._h, u8ptr(x), n, h, w, fptr(pred), u8ptr(rgb), fptr(mins), fptr(maxs)))
        return rgb, mins, maxs, pred

    def infer_clip(self, frames, pass_frames=4, want_depth=False, want_rgb=True, out_rgb=None, out_depth=None):
        """A chunk of the video loop: n frames [n,H,W,3] u8 in passes of `pass_frames`, copies overlapped with compute
        (prisma_depth_infer_stream).  Returns what infer_batch returns.  `frames`/`out_*` from pinned_empty() make the
        host<->device copies asynchronous DMA."""
        x = frames if isinstance(frames, np.ndarray) else np.stack(frames)
        if x.dtype != np.uint8 or x.ndim != 4 or x.shape[3] != 3 or not x.flags.c_contiguous:
            raise PrismaError("expected a C-contiguous [n,H,W,3] uint8 RGB array")
        n, h, w = x.shape[:3]
        pred = (out_depth if out_depth is not None else np.empty((n, h, w), np.float32)) if want_depth else None
        rgb = (out_rgb if out_rgb is not None else np.empty((n, h, w, 3), np.uint8)) if want_rgb else None
        mins = np.empty(n, np.float32)
        maxs = np.empty(n, np.float32)
        check(lib().prisma_depth_infer_stream(self._h, u8ptr(x), n, h, w, pass_frames, fptr(pred), u8ptr(rgb), fptr(mins),
                                              fptr(maxs)))
        return rgb, mins, maxs, pred

    def encode(self, prediction, flip=True):
        """(heat_to_rgb(1 - normalised) * 255).astype(u8) of a given HxW f32 prediction (:215-220)."""
        p = np.ascontiguousarray(prediction, dtype=np.float32)
        h, w = p.shape
        rgb = np.empty((h, w, 3), np.uint8)
        dmin, dmax = C.c_float(), C.c_float()
        check(lib().prisma_depth_encode(self._h, fptr(p), h, w, int(flip), u8ptr(rgb), C.byref(dmin), C.byref(dmax)))
        return rgb, dmin.value, dmax.value

    def encode_png(self, prediction, flip=True):
        """write_depth(normalize, heatmap, encode_range) of a given prediction: the RGB array written to <band>.png."""
        p = np.ascontiguousarray(prediction, dtype=np.float32)
        h, w = p.shape
        rgb = np.empty((h, w, 3), np.uint8)
        dmin, dmax = C.c_float(), C.c_float()
        check(lib().prisma_depth_encode_png(self._h, fptr(p), h, w, int(flip), u8ptr(rgb), C.byref(dmin), C.byref(dmax)))
        return rgb, dmin.value, dmax.value

    def infer_image(self, img, want_depth=True):
        """Still-image path (process_image): (png_rgb u8 HxWx3, min, max, depth f32 HxW | None)."""
        img = np.ascontiguousarray(img)
        if img.dtype != np.uint8 or img.ndim != 3 or img.shape[2] != 3:
            raise PrismaError("expected an HxWx3 uint8 RGB frame")
        h, w = img.shape[:2]
        pred = np.empty((h, w), np.float32) if want_depth else None
        rgb = np.empty((h, w, 3), np.uint8)
        dmin, dmax = C.c_float(), C.c_float()
        check(lib().prisma_depth_infer_image(self._h, u8ptr(img), h, w, fptr(pred), u8ptr(rgb), C.byref(dmin), C.byref(dmax)))
        return rgb, dmin.value, dmax.value, pred

    def point_cloud(self, pred, rgb, flip):
        """write_pcl (bands/common/io.py:201-211) of an HxW f32 prediction and its HxWx3 u8 RGB frame: the H*W vertices
        save_point_cloud writes, as a structured array of PLY_VERTEX_DTYPE (optional flip, 5x5 median, unprojection)."""
        p = np.ascontiguousarray(pred, dtype=np.float32)
        img = np.ascontiguousarray(rgb)
        if p.ndim != 2 or img.dtype != np.uint8 or img.shape != p.shape + (3,):
            raise PrismaError("expected an HxW prediction and an HxWx3 uint8 RGB frame of the same size")
        h, w = p.shape
        out = np.empty(h * w, PLY_VERTEX_DTYPE)
        check(lib().prisma_depth_point_cloud(self._h, fptr(p), h, w, int(bool(flip)), u8ptr(img),
                                             out.ctypes.data_as(c_u8_p)))
        return out

    def read_tap(self, name, shape):
        out = np.empty(int(np.prod(shape)), np.float32)
        n = check(lib().prisma_depth_read_tap(self._h, name.encode(), fptr(out), out.size))
        assert n == out.size, (name, n, out.size)
        return out.reshape(shape)

    def time_resident(self, h, w, iters, batch=1):
        """ms per pass over `batch` resident frames."""
        ms = C.c_float()
        check(lib().prisma_depth_infer_resident(self._h, h, w, batch, iters, C.byref(ms)))
        return ms.value

    def profile(self, h, w, batch=1):
        out = (C.c_float * 8)()
        check(lib().prisma_depth_profile(self._h, h, w, batch, out))
        keys = ["pre", "linear", "attention", "layernorm", "head", "resample", "post", "total"]
        return dict(zip(keys, [float(v) for v in out]))

    def work(self, h, w, batch=1):
        out = (C.c_double * 4)()
        check(lib().prisma_depth_work(self._h, h, w, batch, out))
        return dict(linear_flop=out[0], attention_flop=out[1], head_flop=out[2], launches=int(out[3]))

    def close(self):
        if self._h:
            lib().prisma_engine_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class MidasEngine(DepthAnythingEngine):
    """depth_midas band (bands/depth_midas.py): MiDaS v3 DPT_Large on the same engine -- timm ViT-L/16 encoder with the
    "project" readout at blocks 5/11/17/23, the DPT RefineNet head, bicubic(align_corners=True) to the frame size.
    `state_dict` is the upstream DPTDepthModel checkpoint (dpt_large_384.pt) as is.  `net_side` is the side of the
    transform's fit-inside box: 384 (the hub's default_transform, midas3) or 256 (small_transform, midas3-small)."""

    def __init__(self, state_dict=None, device=0, variant="dpt_large", net_side=384):
        super().__init__(variant, None, device)
        check(lib().prisma_depth_set_net_side(self._h, int(net_side)))
        if state_dict is not None:
            self.load_state_dict(state_dict)


class ZoeDepthEngine(DepthAnythingEngine):
    """depth_anything --metric indoor|outdoor (bands/depth_anything.py:52-57,106-119): the ZoeDepth metric head on the
    Depth-Anything core, fixed 392x518 network input, PIL-bicubic resize of the metric depth to the frame size.
    `state_dict` is depth_anything_metric_depth_{indoor,outdoor}.pt as is (core.core.* + the head)."""

    def __init__(self, state_dict=None, device=0, encoder="vitl"):
        super().__init__("zoe_" + encoder, state_dict, device)
