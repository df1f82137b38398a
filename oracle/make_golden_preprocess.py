"""Regenerate tests/golden/preprocess.pt: frame-sampling indices from the REAL reference function and preprocessing
vectors produced by the reference's own `expand2square` + Pillow's `Image.resize` (the third-party code the reference's
processor calls) + the float ops of transformers 4.40's rescale/normalize.  TEST INFRASTRUCTURE; build container only:
    python -m oracle.make_golden_preprocess"""
from __future__ import annotations

import importlib
import os

import numpy as np
import torch
from PIL import Image

from . import preprocess_ref as P
from . import ref_loader

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "preprocess.pt")
OUT_HD = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "preprocess_hd.pt")

CASES = [   # (name, T, H, W, size, kind, aspect_ratio)
    ("landscape_pad_clip", 3, 90, 160, 56, "clip", "pad"),
    ("portrait_pad_clip", 2, 120, 70, 56, "clip", "pad"),
    ("landscape_nopad_clip", 2, 90, 160, 56, "clip", "resize"),
    ("portrait_nopad_clip", 1, 131, 77, 42, "clip", "resize"),
    ("square_upscale_clip", 1, 20, 20, 56, "clip", "pad"),
    ("landscape_pad_siglip", 2, 72, 128, 70, "siglip", "pad"),
    ("landscape_nopad_siglip", 1, 72, 128, 70, "siglip", "resize"),
    ("hd_pad_clip336", 1, 360, 640, 336, "clip", "pad"),
]


def reference_pipeline(mm_utils, frames, size, kind, aspect_ratio):
    mean = P.SIGLIP_MEAN if kind == "siglip" else P.CLIP_MEAN
    std = P.SIGLIP_STD if kind == "siglip" else P.CLIP_STD
    u8 = []
    for f in frames:
        img = Image.fromarray(f)
        if aspect_ratio == "pad":
            img = mm_utils.expand2square(img, tuple(int(x * 255) for x in mean))     # the reference's own function
        w, h = img.size
        oh, ow = P.resize_target(h, w, size, kind)
        img = img.resize((ow, oh), resample=Image.BICUBIC)                           # transformers 4.40 resize -> PIL
        arr = np.array(img)
        if kind != "siglip":
            top, left = (oh - size) // 2, (ow - size) // 2
            arr = arr[top:top + size, left:left + size]
        u8.append(arr)
    u8 = np.stack(u8)
    x = (u8 * (1 / 255)).astype(np.float32)                                           # rescale
    x = (x - np.array(mean, dtype=np.float32)) / np.array(std, dtype=np.float32)      # normalize (channels last)
    return u8, np.ascontiguousarray(x.transpose(0, 3, 1, 2))


def save_deflated(obj, path):
    """torch.save, then the archive's members deflated (torch.load reads either form): the uint8 frames are mostly smooth."""
    import io
    import zipfile
    buf = io.BytesIO()
    torch.save(obj, buf)
    with zipfile.ZipFile(io.BytesIO(buf.getvalue())) as zi, zipfile.ZipFile(path, "w", zipfile.ZIP_DEFLATED, compresslevel=9) as zo:
        for info in zi.infolist():
            zo.writestr(info.filename, zi.read(info.filename))


def main():
    ref_loader.load()
    mm_utils = importlib.import_module("videollama2.mm_utils")
    out = {"frame_sample": [], "cases": {}}
    for duration in (1, 2, 7, 8, 9, 16, 31, 100, 257, 1000, 5400):
        for n in (1, 8, 16, 32):
            out["frame_sample"].append(("uniform", duration, n, None, mm_utils.frame_sample(duration, "uniform", num_frames=n).tolist()))
        for fps in (1, 3, 24.0, 25, 29.97, 30.0, 60):
            out["frame_sample"].append(("fps", duration, None, fps, mm_utils.frame_sample(duration, "fps", fps=fps).tolist()))
    rng = np.random.default_rng(20240604)
    for name, T, H, W, size, kind, ar in CASES:
        # smooth random content + sharp edges + saturated regions (exercise the negative bicubic lobes and the clipping)
        base = rng.integers(0, 256, (T, H // 6 + 2, W // 6 + 2, 3), dtype=np.uint8)
        frames = np.stack([np.array(Image.fromarray(b).resize((W, H), Image.BILINEAR)) for b in base])
        frames[:, : H // 4, : W // 3] = 255
        frames[:, H // 2:, W // 2: W // 2 + 3] = 0
        frames[:, ::7, ::5] = rng.integers(0, 256, frames[:, ::7, ::5].shape, dtype=np.uint8)
        u8, px = reference_pipeline(mm_utils, frames, size, kind, ar)
        out["cases"][name] = {"T": T, "H": H, "W": W, "size": size, "kind": kind, "aspect_ratio": ar,
                              "frames": torch.from_numpy(frames), "u8": torch.from_numpy(u8),
                              # float32 pixel_values only for the small cases (fixture size); u8 -> float is a 256-entry map
                              "pixel_values": torch.from_numpy(px) if size <= 70 else None}
    # the HD case goes to a file of its own: every committed fixture stays under 1 MB
    hd = {"cases": {k: out["cases"].pop(k) for k in list(out["cases"]) if out["cases"][k]["H"] * out["cases"][k]["W"] >= 360 * 640}}
    for path, obj in ((OUT, out), (OUT_HD, hd)):
        save_deflated(obj, path)
        print("wrote", path, os.path.getsize(path) // 1024, "KiB")


if __name__ == "__main__":
    main()
