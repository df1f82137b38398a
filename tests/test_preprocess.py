"""Frame preprocessing (SURVEY.md §8f row 3): the numpy oracle against Pillow itself and the committed goldens, the
product's host tables against the oracle's, frame_sample against the reference's outputs; on the GPU the CUDA resampler
must reproduce Pillow's uint8 image bit for bit and the bf16 pixel_values must be the bf16 rounding of the reference's
float32 values, and the fp16 pixel_values (the reference calls .half() on them) its fp16 rounding."""
import os

import numpy as np
import pytest
import torch

from test_kernels_exact_gpu import storage_params

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "preprocess.pt")
GOLD_HD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "preprocess_hd.pt")   # the 640 x 360 case


@pytest.fixture(scope="module")
def gold():
    g = torch.load(GOLD)
    g["cases"].update(torch.load(GOLD_HD)["cases"])
    return g


def test_oracle_resample_matches_pillow_live():
    Image = pytest.importorskip("PIL.Image")
    from oracle import preprocess_ref as P
    rng = np.random.default_rng(1)
    for h, w, oh, ow in [(48, 64, 33, 44), (108, 192, 34, 34), (10, 10, 34, 34), (34, 50, 34, 50), (37, 53, 20, 90),
                         (64, 64, 34, 34), (7, 9, 3, 4), (200, 31, 17, 31)]:
        img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        ref = np.array(Image.fromarray(img).resize((ow, oh), resample=Image.BICUBIC))
        assert np.array_equal(P.resample_u8(img, oh, ow), ref), (h, w, oh, ow)


def test_oracle_matches_goldens(gold):
    from oracle import preprocess_ref as P
    for name, c in gold["cases"].items():
        u8, px = P.preprocess_frames(list(c["frames"].numpy()), c["size"], c["kind"], c["aspect_ratio"])
        assert np.array_equal(u8, c["u8"].numpy()), name                      # integer work: bit-exact
        if c["pixel_values"] is not None:
            assert np.array_equal(px, c["pixel_values"].numpy()), name       # same float32 ops in the same order


def test_host_tables_and_geometry_match_oracle(gold):
    from oracle import preprocess_ref as P
    from videollama2_b200 import preprocess as pp
    for n_in, n_out in [(1920, 336), (640, 336), (336, 336), (20, 56), (131, 71), (1080, 384), (77, 42)]:
        b0, k0, ks0 = P.pil_coeffs(n_in, n_out)
        b1, k1, ks1 = pp.resample_tables(n_in, n_out)
        assert ks0 == ks1 and np.array_equal(b0, b1) and np.array_equal(k0, k1)
    assert np.array_equal(pp.normalise_lut(P.CLIP_MEAN, P.CLIP_STD), P.normalise_lut(P.CLIP_MEAN, P.CLIP_STD))
    for h, w, size, kind in [(90, 160, 56, "clip"), (131, 77, 42, "clip"), (72, 128, 70, "siglip"), (50, 50, 56, "clip")]:
        for ar in ("pad", "resize"):
            ch, cw, oy, ox, oh, ow, ct, cl = pp.geometry(h, w, size, kind, ar)
            sq = P.expand2square(np.zeros((h, w, 3), np.uint8), (1, 2, 3)) if ar == "pad" else np.zeros((h, w, 3), np.uint8)
            assert (ch, cw) == sq.shape[:2]
            assert (oh, ow) == P.resize_target(ch, cw, size, kind)
            if kind == "clip":
                assert (ct, cl) == ((oh - size) // 2, (ow - size) // 2)
    # an identity axis (in == out) is the identity in fixed point, which is why Pillow may skip the pass
    b, k, ks = pp.resample_tables(40, 40)
    for xx in range(40):
        taps = {int(b[xx, 0]) + j: int(k[xx, j]) for j in range(int(b[xx, 1])) if k[xx, j]}
        assert taps == {xx: 1 << 22}


def test_frame_sample_matches_reference(gold):
    from videollama2_b200 import mm_utils
    for mode, duration, n, fps, want in gold["frame_sample"]:
        got = mm_utils.frame_sample(duration, mode, num_frames=n, fps=fps)
        assert got.tolist() == want, (mode, duration, n, fps)
    with pytest.raises(ImportError):
        mm_utils.frame_sample(10, "random")


def test_preprocess_refuses_cpu_tensors():
    from videollama2_b200 import preprocess as pp
    from videollama2_b200._lib import Vl2Error
    with pytest.raises(Vl2Error):
        pp.preprocess_frames(torch.zeros((1, 8, 8, 3), dtype=torch.uint8), 4, (0.5,) * 3, (0.5,) * 3)


class _Proc:
    def __init__(self, kind, size):
        from oracle import preprocess_ref as P
        if kind == "siglip":
            self.size = {"height": size, "width": size}
            self.image_mean, self.image_std = list(P.SIGLIP_MEAN), list(P.SIGLIP_STD)
        else:
            self.size = {"shortest_edge": size}
            self.image_mean, self.image_std = list(P.CLIP_MEAN), list(P.CLIP_STD)
        self.crop_size = {"height": size, "width": size}


@pytest.mark.gpu
def test_gpu_preprocess_matches_goldens(gold, cuda):
    _preprocess_matches_goldens(gold, cuda, torch.bfloat16)


@pytest.mark.gpu
def test_gpu_preprocess_matches_goldens_fp16(gold, cuda):
    """fp16 pixel_values (the reference calls .half() on them): the fp16 rounding of the goldens' float32 values."""
    _preprocess_matches_goldens(gold, cuda, torch.float16)


def _preprocess_matches_goldens(gold, cuda, dt):
    from videollama2_b200 import preprocess as pp
    for name, c in gold["cases"].items():
        proc = _Proc(c["kind"], c["size"])
        out, u8 = pp.preprocess_frames(c["frames"].to(cuda), c["size"], proc.image_mean, proc.image_std, kind=c["kind"],
                                       aspect_ratio=c["aspect_ratio"], return_u8=True, dtype=dt)
        assert torch.equal(u8.cpu(), c["u8"]), name                              # Pillow's uint8 image, bit for bit
        assert out.shape == (c["T"], 3, c["size"], c["size"]) and out.dtype == dt
        if c["pixel_values"] is not None:
            assert torch.equal(out.cpu(), c["pixel_values"].to(dt)), name


@pytest.mark.gpu
@storage_params("H,W,size,kind,ar", [(1080, 1920, 336, "clip", "pad"), (720, 1280, 384, "siglip", "pad"),
                                     (480, 854, 336, "clip", "resize"), (1920, 1080, 336, "clip", "pad"),
                                     (336, 336, 336, "clip", "pad"), (100, 60, 336, "clip", "pad")])
def test_gpu_preprocess_full_size_vs_oracle(cuda, dt, H, W, size, kind, ar):
    """Real frame sizes against the numpy oracle (which is pinned to Pillow above), bf16 and fp16 pixel_values."""
    from oracle import preprocess_ref as P
    from videollama2_b200 import preprocess as pp
    rng = np.random.default_rng(H * 7 + W)
    small = rng.integers(0, 256, (2, H // 8 + 1, W // 8 + 1, 3), dtype=np.uint8)
    frames = np.repeat(np.repeat(small, 8, axis=1), 8, axis=2)[:, :H, :W].copy()
    frames[:, ::3, ::11] = rng.integers(0, 256, frames[:, ::3, ::11].shape, dtype=np.uint8)
    proc = _Proc(kind, size)
    ref_u8, ref_px = P.preprocess_frames(list(frames), size, kind, ar)
    out, u8 = pp.preprocess_frames(torch.from_numpy(frames).to(cuda), size, proc.image_mean, proc.image_std, kind=kind,
                                   aspect_ratio=ar, return_u8=True, dtype=dt)
    assert np.array_equal(u8.cpu().numpy(), ref_u8)
    assert out.dtype == dt and torch.equal(out.cpu(), torch.from_numpy(ref_px).to(dt))


@pytest.mark.gpu
def test_process_video_semantics(cuda):
    """mm_utils.process_video on decoded frames: short clips are padded with black frames whose width/height are swapped
    like the reference's `np.zeros((*pil.size, 3))`, at most MAX_FRAMES are kept, tensors and lists agree."""
    from oracle import preprocess_ref as P
    from videollama2_b200 import mm_utils
    rng = np.random.default_rng(3)
    frames = rng.integers(0, 256, (3, 40, 64, 3), dtype=np.uint8)
    proc = _Proc("clip", 28)
    out = mm_utils.process_video(frames, proc, num_frames=5, device=cuda)
    assert out.shape == (5, 3, 28, 28)
    # each appended black frame takes (*previous.size, 3) = (width, height, 3): the shapes alternate
    black = [np.zeros((64, 40, 3), np.uint8), np.zeros((40, 64, 3), np.uint8)]
    _, ref = P.preprocess_frames(list(frames) + black, 28, "clip", "pad")
    assert torch.equal(out.cpu(), torch.from_numpy(ref).to(torch.bfloat16))
    same = mm_utils.process_video(torch.from_numpy(frames).to(cuda), proc, num_frames=3, device=cuda)
    assert torch.equal(same, out[:3])
    many = mm_utils.process_video(np.repeat(frames, 14, axis=0), proc, num_frames=8, device=cuda)
    assert many.shape[0] == 32                                                   # MAX_FRAMES
    img = mm_utils.process_image(frames[0], proc, device=cuda)
    assert img.shape == (1, 3, 28, 28) and torch.equal(img[0], out[0])
    with pytest.raises(NotImplementedError):
        mm_utils.process_video("clip.mp4", proc)
