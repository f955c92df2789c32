"""CPU oracle: depth_midas --model midas3-small (TEST INFRASTRUCTURE ONLY, see oracle/__init__.py).

midas3-small is the DPT_Large network of oracle/midas.py behind the hub's small_transform instead of its default_transform
(bands/depth_midas.py:39-42).  The two transforms differ only in the side of the fit-inside box: Resize(256, 256, keep AR,
x32, "upper_bound", INTER_CUBIC) instead of 384, with the same ImageNet statistics and PrepareForNet.  Parity unpinned, as
for oracle/midas.py: the hub code is not vendored and this is restated from the published intel-isl/MiDaS hubconf.py.
"""
import cv2
import numpy as np
import torch
import torch.nn.functional as F

from .da import _ident
from .midas import midas_get_size, midas_model

SMALL_SIDE = 256


def midas_small_preprocess(img_u8, target=SMALL_SIDE):
    """small_transform: /255 (f64), Resize(target, target, keep AR, x32, "upper_bound", INTER_CUBIC), NormalizeImage(ImageNet
    mean / std), PrepareForNet (CHW f32).  target=384 is oracle.midas.midas_preprocess (default_transform)."""
    image = img_u8 / 255.0
    w, h = midas_get_size(image.shape[1], image.shape[0], target)
    image = cv2.resize(image, (w, h), interpolation=cv2.INTER_CUBIC)
    image = (image - np.array([0.485, 0.456, 0.406])) / np.array([0.229, 0.224, 0.225])
    return np.ascontiguousarray(np.transpose(image, (2, 0, 1))).astype(np.float32)


def midas_small_infer(sd, img_u8, variant="dpt_large", q=_ident, target=SMALL_SIDE):
    """infer(img, model_version="midas3-small") (bands/depth_midas.py:49-75): small_transform -> model ->
    bicubic(align_corners=True) to the frame size -> f32 HxW."""
    x = torch.from_numpy(midas_small_preprocess(img_u8, target)).unsqueeze(0)
    with torch.no_grad():
        pred = midas_model(sd, x, variant, q)
        pred = F.interpolate(pred.unsqueeze(1), size=img_u8.shape[:2], mode="bicubic", align_corners=True).squeeze()
    return pred.numpy().astype(np.float32)
