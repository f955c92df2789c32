"""Container I/O for the band scripts (reference: bands/common/io.py VideoWriter :246-305, decord readers).

Codec work is OUT OF SCOPE of the H100 engine (SURVEY.md section 2: CPU codec, lossy).  The reference uses decord +
PyAV/libx264, neither of which is installed in this image; OpenCV's capture/writer is, and is used here.  Frames
cross this boundary as HxWx3 uint8 RGB arrays, exactly what the reference's loops hand to infer().
"""
import os

import cv2
import numpy as np


class VideoReader:
    def __init__(self, path):
        self.cap = cv2.VideoCapture(path)
        if not self.cap.isOpened():
            raise IOError(f"cannot open video {path}")
        self.width = int(self.cap.get(cv2.CAP_PROP_FRAME_WIDTH))
        self.height = int(self.cap.get(cv2.CAP_PROP_FRAME_HEIGHT))
        self.fps = float(self.cap.get(cv2.CAP_PROP_FPS)) or 24.0
        self.frames = int(self.cap.get(cv2.CAP_PROP_FRAME_COUNT))

    def __len__(self):
        return self.frames

    def __iter__(self):
        while True:
            ok, bgr = self.cap.read()
            if not ok:
                return
            yield np.ascontiguousarray(bgr[..., ::-1])

    def get_avg_fps(self):
        return self.fps

    def seek(self, index):
        """Next frame returned by the iterator = frame `index` (a frame-range worker starts mid-clip).  OpenCV seeks to the
        preceding key frame and decodes forward; the position is verified, and if the container's index is inexact (B-frame
        streams) the reader falls back to decoding from the first frame and discarding."""
        index = int(index)
        self.cap.set(cv2.CAP_PROP_POS_FRAMES, index)
        if int(round(self.cap.get(cv2.CAP_PROP_POS_FRAMES))) != index:
            self.cap.set(cv2.CAP_PROP_POS_FRAMES, 0)
            for _ in range(index):
                if not self.cap.grab():
                    break


class VideoWriter:
    def __init__(self, width, height, frame_rate, filename):
        self.size = (int(width), int(height))
        self.w = cv2.VideoWriter(filename, cv2.VideoWriter_fourcc(*"mp4v"), float(frame_rate), self.size)
        if not self.w.isOpened():
            raise IOError(f"cannot open video writer for {filename}")

    def write(self, rgb):
        if (rgb.shape[1], rgb.shape[0]) != self.size:  # the reference rescales inside libswscale (io.py:296-297)
            rgb = cv2.resize(rgb, self.size, interpolation=cv2.INTER_LINEAR)
        self.w.write(np.ascontiguousarray(rgb[..., ::-1]))

    def close(self):
        self.w.release()


def open_rgb(path):
    bgr = cv2.imread(path, cv2.IMREAD_COLOR)
    if bgr is None:
        raise IOError(f"cannot read image {path}")
    return np.ascontiguousarray(bgr[..., ::-1])


def write_rgb(path, rgb):
    cv2.imwrite(path, np.ascontiguousarray(rgb[..., ::-1]))


def create_folder(path):
    os.makedirs(path, exist_ok=True)
