"""Host-side mirror of the reference mask band interface (bands/mask_mmdet.py) on top of the C ABI.

`SoloV2Engine(state_dict)` ≙ `init_detector(CONFIG, MODEL)` (mask_mmdet.py:38-41); `infer(rgb)` ≙
`inference_detector(model, img)` (apis/inference.py:99-162) plus the band's union loop (mask_mmdet.py:43-61,134-146);
`inference_detector(rgb)` returns the reference's (bbox_results, mask_results) structure
(models/detectors/single_stage_instance_seg.py:184-250).  All arithmetic happens in libprisma_b200.so.
"""
import ctypes as C

import numpy as np

from ._lib import PrismaError, check, fptr, lib, u8ptr, c_i64_p

CLASSES = ['person', 'bird', 'cat', 'dog', 'horse', 'sheep', 'cow', 'elephant', 'bear', 'zebra', 'giraffe']  # mask_mmdet.py:29
NUM_CLASSES = 80
MAX_PER_IMG = 100


def sdf_green(union, device=0):
    """getSDF (bands/mask_mmdet.py:64-69) of an HxW u8 union mask -> the HxW u8 green channel written with --sdf."""
    union = np.ascontiguousarray(union, dtype=np.uint8)
    if union.ndim != 2:
        raise PrismaError("expected an HxW uint8 mask")
    out = np.empty_like(union)
    check(lib().prisma_mask_sdf(device, u8ptr(union), union.shape[0], union.shape[1], u8ptr(out)))
    return out


class SoloV2Engine:
    def __init__(self, state_dict=None, device=0, variant="r101"):
        self._h = C.c_void_p()
        check(lib().prisma_mask_create(variant.encode(), device, C.byref(self._h)))
        if state_dict is not None:
            self.load_state_dict(state_dict)

    def load_state_dict(self, state_dict):
        l = lib()
        for name, t in state_dict.items():
            a = t.detach().cpu().numpy() if hasattr(t, "detach") else np.asarray(t)
            if a.dtype.kind != "f":
                continue  # num_batches_tracked
            a = np.ascontiguousarray(a, dtype=np.float32)
            shape = (C.c_int64 * max(a.ndim, 1))(*(a.shape if a.ndim else (1,)))
            check(l.prisma_mask_load_tensor(self._h, name.encode(), fptr(a), C.cast(shape, c_i64_p), max(a.ndim, 1)))
        check(l.prisma_mask_finalize(self._h))

    def infer(self, rgb, confidence=0.5, want_instances=False):
        """HxWx3 u8 RGB -> dict(union HxW u8, scores [n], labels [n], masks [n,H,W] bool | None, ms)."""
        rgb = np.ascontiguousarray(rgb)
        if rgb.dtype != np.uint8 or rgb.ndim != 3 or rgb.shape[2] != 3:
            raise PrismaError("expected an HxWx3 uint8 RGB frame")
        h, w = rgb.shape[:2]
        union = np.empty((h, w), np.uint8)
        scores = np.zeros(MAX_PER_IMG, np.float32)
        labels = np.zeros(MAX_PER_IMG, np.int32)
        inst = np.empty((MAX_PER_IMG, h, w), np.uint8) if want_instances else None
        n, ms = C.c_int(), C.c_float()
        check(lib().prisma_mask_infer(self._h, u8ptr(rgb), h, w, float(confidence), u8ptr(union), C.byref(n), fptr(scores),
                                      labels.ctypes.data_as(C.POINTER(C.c_int32)), u8ptr(inst), C.byref(ms)))
        k = n.value
        return dict(union=union, scores=scores[:k].copy(), labels=labels[:k].copy(),
                    masks=inst[:k].astype(bool) if want_instances else None, ms=ms.value)

    def infer_from_feats(self, feats, frame_hw, confidence=0.5, want_instances=True, img_shape=None):
        """Tests: head + decode replayed from five given FPN levels (each [1|,256,h,w] float32, NCHW) for a frame of size
        frame_hw whose plan exists (call infer once on a frame of that size).  img_shape = the (h, w) of the resized image the
        reference's meta carried (default: the engine's own test-pipeline size).  Same result dict as infer()."""
        ih, iw = img_shape if img_shape is not None else (0, 0)
        h, w = frame_hw
        for lvl, f in enumerate(feats):
            f = np.ascontiguousarray(np.asarray(f, np.float32).reshape(256, f.shape[-2], f.shape[-1]))
            check(lib().prisma_mask_inject_feat(self._h, lvl, fptr(f), f.shape[1], f.shape[2]))
        union = np.empty((h, w), np.uint8)
        scores = np.zeros(MAX_PER_IMG, np.float32)
        labels = np.zeros(MAX_PER_IMG, np.int32)
        inst = np.empty((MAX_PER_IMG, h, w), np.uint8) if want_instances else None
        n = C.c_int()
        check(lib().prisma_mask_infer_from_feats(self._h, h, w, int(ih), int(iw), float(confidence), u8ptr(union), C.byref(n), fptr(scores),
                                                 labels.ctypes.data_as(C.POINTER(C.c_int32)), u8ptr(inst)))
        k = n.value
        return dict(union=union, scores=scores[:k].copy(), labels=labels[:k].copy(),
                    masks=inst[:k].astype(bool) if want_instances else None)

    def inference_detector(self, rgb):
        """(bbox_results, mask_results) as the reference's format_results: 80 arrays (n,5) [0,0,0,0,score] and 80 lists of
        HxW bool masks."""
        r = self.infer(rgb, want_instances=True)
        bbox = [np.zeros((0, 5), np.float32) for _ in range(NUM_CLASSES)]
        masks = [[] for _ in range(NUM_CLASSES)]
        for c in range(NUM_CLASSES):
            sel = r["labels"] == c
            if sel.any():
                b = np.zeros((int(sel.sum()), 5), np.float32)
                b[:, 4] = r["scores"][sel]
                bbox[c] = b
                masks[c] = [m for m in r["masks"][sel]]
        return bbox, masks

    def read_tap(self, name, shape):
        out = np.empty(int(np.prod(shape)), np.float32)
        n = check(lib().prisma_mask_read_tap(self._h, name.encode(), fptr(out), out.size))
        assert n == out.size, (name, n, out.size)
        return out.reshape(shape)

    def work(self, h, w):
        out = (C.c_double * 8)()
        check(lib().prisma_mask_work(self._h, h, w, out))
        return dict(flop=out[0], launches=int(out[1]), resized=(int(out[2]), int(out[3])), padded=(int(out[4]), int(out[5])))

    def close(self):
        if self._h:
            lib().prisma_engine_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class SoloV2Lanes:
    """The video loop of the band (mask_mmdet.py:131-154) over several engines at once: frames are independent, so `lanes`
    engines (one handle, stream, CUDA graph and set of plan buffers each; a handle is not re-entrant) take consecutive frames
    from worker threads -- the C calls release the GIL -- and the GPU overlaps the passes: one frame's ~200 short launches no
    longer leave the SMs idle between kernels.  Results come back in frame order and are the same as SoloV2Engine.infer's."""

    def __init__(self, state_dict, device=0, variant="r101", lanes=4):
        from concurrent.futures import ThreadPoolExecutor
        self.engines = [SoloV2Engine(state_dict, device=device, variant=variant) for _ in range(max(1, int(lanes)))]
        self._pool = ThreadPoolExecutor(max_workers=len(self.engines))

    def infer(self, rgb, **kw):
        return self.engines[0].infer(rgb, **kw)

    def map(self, frames, confidence=0.5, want_instances=False):
        """frames: iterable of HxWx3 u8 RGB -> generator of infer() dicts, in order; at most `lanes` frames are in flight."""
        import collections
        free = collections.deque(self.engines)
        pending = collections.deque()   # (future, engine)

        def run(eng, f):
            return eng.infer(f, confidence=confidence, want_instances=want_instances)
        for f in frames:
            if not free:
                fut, eng = pending.popleft()
                r = fut.result()
                free.append(eng)
                yield r
            eng = free.popleft()
            pending.append((self._pool.submit(run, eng, f), eng))
        while pending:
            fut, eng = pending.popleft()
            r = fut.result()
            free.append(eng)
            yield r

    def close(self):
        self._pool.shutdown(wait=True)
        for e in self.engines:
            e.close()
