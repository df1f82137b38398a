"""Programmatic dependent launch (PDL) gives the same bits as ordinary stream order.  Every case runs on the bf16 and the
fp16 build (the `dt` parameter) and compares bit for bit with the same sequence run with PDL off.

a. Read after write.  The producer is a slow GEMM launched under PDL: it releases its dependents at its first
   instruction, then runs for about a millisecond on four SMs (four 128 x 256 tiles, K = 131072: ~8.6 GFLOP per tile,
   several hundred times a consumer's run time).  Its operands make the output exact, A = [I | 0] and W = [D^T | 0] give
   C = D, so it writes any chosen tensor, of the storage type or fp32, as the consumer's input.  The consumer is launched
   right after it, also under PDL; a consumer that read before its griddepcontrol.wait would see C's previous contents
   (zeros).  Everything is allocated up front, and nothing but the consumer's own launches (torch.empty allocates, it
   launches nothing) sits between the two: a torch fill, copy or .contiguous() in between would end the programmatic
   edge and the probe would prove nothing.  One probe has the decode GEMV as its producer, which releases its dependents
   after its k-loop but before its stores (the tensor-parallel decode step: GEMV, then the all-reduce).
b. Write after read.  The consumer's output aliases the last k-blocks of the slow GEMM's A, which the GEMM reads last.
   A is zero there and W is all ones, so C is still exactly D, and a consumer that wrote before its wait would change C.
c. The engine: graph-replayed greedy, sampled and processed decoding with decode_pdl on and off, the captured decode graph's
   programmatic edges, eager encode / prefill / preprocessing under ops.pdl(True), and nested ops.pdl blocks.

A consumer that does not wait shows up as wrong values, never as a fault: the all-reduce probe gives every call a fresh
zeroed signal pad and epoch 1, which its start and end barriers pass on one GPU."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

from helpers import build_engine

pytestmark = pytest.mark.gpu
DTYPES = [torch.bfloat16, torch.float16]
DT_IDS = ["bf16", "fp16"]
M, N, K = 128, 1024, 131072          # four 128 x 256 tiles (bn = 256 forced), each one SM for ~1 ms
TAIL = 8192                          # W's last k-blocks are ones (A is zero there): the write-after-read probes' target


def _abi(dt, name, *args):
    from videollama2_b200 import _lib
    lib = _lib.load(dt)
    _lib.check(getattr(lib, name)(*args, torch.cuda.current_stream().cuda_stream), name, lib)


def _bits(t):
    t = t.detach().contiguous()
    return t.view(torch.uint8) if t.dtype != torch.bool else t


def _same(a, b):
    return a.shape == b.shape and torch.equal(_bits(a), _bits(b))


def _wrong(a, b):
    """Elements of a whose bits differ from b's."""
    if a.element_size() == 1:
        return int((a != b).sum())
    iv = {2: torch.int16, 4: torch.int32, 8: torch.int64}[a.element_size()]
    return int((a.contiguous().view(iv) != b.contiguous().view(iv)).sum())


class Slow:
    """The slow producer: ops.gemm(A, W) = D into out (storage type [M, N] or fp32 [M, N])."""

    def __init__(self, dt, dev):
        self.dt, self.dev = dt, dev
        self.A = torch.zeros((M, K), device=dev, dtype=dt)
        self.A[:, :M] = torch.eye(M, device=dev, dtype=dt)
        self.W = torch.zeros((N, K), device=dev, dtype=dt)
        self.W[:, K - TAIL:] = 1
        self.out = torch.zeros((M, N), device=dev, dtype=dt)
        self.out32 = torch.zeros((M, N), device=dev, dtype=torch.float32)
        g = torch.Generator(device="cpu").manual_seed(1)
        self.D = (torch.randn((M, N), generator=g) * 2).to(dt).to(dev)     # finite and non-zero: C = D exactly
        self.W[:, :M] = self.D.t()

    def arm(self):
        """Before a probe (outside its launch pair): C back to zeros, A's tail back to zeros."""
        self.out.zero_()
        self.out32.zero_()
        self.A[:, K - TAIL:] = 0

    def launch(self, f32=False):
        from videollama2_b200 import ops
        return ops.gemm(self.A, self.W, out=self.out32 if f32 else self.out, bn=256, splitk=False)

    def tail(self, nbytes):
        """The last nbytes of A (the end of its last row): read by the GEMM in its final k-blocks."""
        assert nbytes <= TAIL * self.A.element_size()
        return self.A.view(-1).view(torch.uint8)[-nbytes:]


@pytest.fixture(scope="module", params=DTYPES, ids=DT_IDS)
def slow(request, cuda):
    s = Slow(request.param, cuda)
    s.arm()
    s.launch()
    torch.cuda.synchronize()
    assert torch.equal(s.out, s.D)
    yield s
    del s
    torch.cuda.empty_cache()


def run_pair(slow, consumer, f32=False):
    """The producer and the consumer with PDL off, then on.  Returns ((outputs off, C off), (outputs on, C on))."""
    from videollama2_b200 import ops
    res = []
    for on in (False, True):
        slow.arm()
        run = consumer()           # allocates and prepares everything; returns the launch closure
        torch.cuda.synchronize()
        with ops.pdl(on):
            slow.launch(f32)
            outs = run()
        torch.cuda.synchronize()
        res.append(([o.clone() for o in outs], (slow.out32 if f32 else slow.out).clone()))
    return res


def check_raw(slow, consumer, f32=False, what="", inplace=False):
    """`inplace`: the consumer edits the producer's output (compared as one of its outputs instead)."""
    (off, c_off), (on, c_on) = run_pair(slow, consumer, f32)
    want = slow.D.float() if f32 else slow.D
    assert inplace or (_same(c_off, want) and _same(c_on, want)), f"{what}: the producer's output is not D"
    for i, (a, b) in enumerate(zip(on, off)):
        assert _same(a, b), f"{what}: output {i} differs under PDL in {_wrong(a, b)} of {a.numel()} elements"
    return off


# ---------------------------------------------------------------------------------------------------------------------
# a. read after write
# ---------------------------------------------------------------------------------------------------------------------
def _preprocess_args(dt, dev, frames, tmp=None):
    """vl2_preprocess_args for 1 x 40 x 64 frames -> 28 x 28 (CLIP, padded to a square); tmp and outputs allocated."""
    from videollama2_b200 import _lib, preprocess as pp
    from oracle import preprocess_ref as P
    T, H, W, _ = frames.shape
    ch, cw, oy, ox, out_h, out_w, ctop, cleft = pp.geometry(H, W, 28, "clip", "pad")
    bh, kh, ksh = pp._tables_on(dev, cw, out_w)
    bv, kv, ksv = pp._tables_on(dev, ch, out_h)
    keep = {"lut": torch.from_numpy(pp.normalise_lut(P.CLIP_MEAN, P.CLIP_STD)).to(dev),
            "out": torch.empty((T, 3, 28, 28), device=dev, dtype=dt),
            "u8": torch.empty((T, 28, 28, 3), device=dev, dtype=torch.uint8), "tables": (bh, kh, bv, kv)}
    a = pp.PreprocessArgs()
    a.frames, a.T, a.H, a.W = frames.data_ptr(), T, H, W
    a.canvas_h, a.canvas_w, a.off_y, a.off_x = ch, cw, oy, ox
    for i, v in enumerate(int(x * 255) for x in P.CLIP_MEAN):
        a.pad_rgb[i] = v
    a.out_h, a.out_w, a.crop_top, a.crop_left, a.crop = out_h, out_w, ctop, cleft, 28
    a.bounds_h, a.kk_h, a.ksize_h = bh.data_ptr(), kh.data_ptr(), ksh
    a.bounds_v, a.kk_v, a.ksize_v = bv.data_ptr(), kv.data_ptr(), ksv
    a.lut = keep["lut"].data_ptr()
    nbytes = int(_lib.load(dt).vl2_preprocess_workspace(C.byref(a)))
    if tmp is None:
        tmp = torch.empty((nbytes,), device=dev, dtype=torch.uint8)
    assert tmp.numel() >= nbytes
    keep["tmp"] = tmp
    a.tmp, a.out_bf16, a.out_u8 = tmp.data_ptr(), keep["out"].data_ptr(), keep["u8"].data_ptr()
    return a, keep


def test_preprocess_reads_frames_after_the_producer(slow, cuda):
    """The frames are D's bytes: 1 x 40 x 64 x 3 uint8 (7680 bytes of the producer's output)."""
    frames = slow.out.view(-1).view(torch.uint8)[:40 * 64 * 3].view(1, 40, 64, 3)

    def consumer():
        a, keep = _preprocess_args(slow.dt, cuda, frames)

        def run():
            _abi(slow.dt, "vl2_preprocess_frames", C.byref(a))
            return [keep["u8"], keep["out"]]
        return run
    off = check_raw(slow, consumer, what="vl2_preprocess_frames")
    # and it is the preprocessing of D's bytes
    from videollama2_b200 import preprocess as pp
    from oracle import preprocess_ref as P
    want = pp.preprocess_frames(slow.D.view(-1).view(torch.uint8)[:40 * 64 * 3].view(1, 40, 64, 3).clone(), 28,
                                P.CLIP_MEAN, P.CLIP_STD, return_u8=True, dtype=slow.dt)
    assert _same(off[0], want[1]) and _same(off[1], want[0])


def _allreduce(dt, part, xout, stats, pad, S, H):
    from videollama2_b200 import _lib
    a = _lib.TpAllReduceArgs()
    a.part[0], a.xout[0], a.stats[0], a.pads[0] = part.data_ptr(), xout.data_ptr(), stats.data_ptr(), pad.data_ptr()
    a.rank, a.world, a.S, a.H, a.epoch, a.inswitch_reduce = 0, 1, S, H, 1, 0
    _abi(dt, "vl2_tp_allreduce_stats", C.byref(a))


def _allreduce_consumer(dt, dev, part, S, H):
    def consumer():
        xout = torch.empty((S, H), device=dev, dtype=dt)
        stats = torch.empty((S,), device=dev, dtype=torch.float32)
        pad = torch.zeros((32,), device=dev, dtype=torch.int32)     # fresh pad, epoch 1: the barriers pass on one GPU

        def run():
            _allreduce(dt, part, xout, stats, pad, S, H)
            return [xout, stats]
        return run
    return consumer


def _check_allreduce(off, D):
    xout, stats = off
    assert _same(xout, D)
    ref = D.double().pow(2).sum(1)
    # fp32 fma accumulation over H products plus the block reduction: relative error below (H + 8) 2^-24
    assert torch.allclose(stats.double(), ref, rtol=(D.shape[1] + 8) * 2.0 ** -24, atol=0)


def test_allreduce_reads_partials_after_the_producer(slow, cuda):
    """vl2_tp_allreduce_stats with world = 1: part[0] = D ([128, 1024]); xout must be D, stats its fp64 row sums of
    squares."""
    off = check_raw(slow, _allreduce_consumer(slow.dt, cuda, slow.out, M, N), what="vl2_tp_allreduce_stats")
    _check_allreduce(off, slow.D)


def test_allreduce_after_the_gemv(cuda, dt):
    """The decode GEMV releases its dependents after its k-loop, before its stores: y = W e0 = column 0 of W."""
    from videollama2_b200 import ops
    S, H, Kg = 4, 2048, 4096
    g = torch.Generator(device="cpu").manual_seed(2)
    D = (torch.randn((S * H,), generator=g) * 2).to(dt).to(cuda)
    W = torch.zeros((S * H, Kg), device=cuda, dtype=dt)
    W[:, 0] = D
    x = torch.zeros((Kg,), device=cuda, dtype=dt)
    x[0] = 1
    y = torch.zeros((1, S * H), device=cuda, dtype=dt)
    res = []
    for on in (False, True):
        y.zero_()
        run = _allreduce_consumer(dt, cuda, y, S, H)()
        gamma = torch.ones((H,), device=cuda, dtype=dt)
        torch.cuda.synchronize()
        with ops.pdl(on):
            ops.gemv(x, W, out=y)
            outs = run() + [ops.rmsnorm(y.view(S, H), gamma, 1e-5)]
        torch.cuda.synchronize()
        res.append([o.clone() for o in outs])
    assert _same(res[0][0], D.view(S, H))
    for i, (a, b) in enumerate(zip(res[1], res[0])):
        assert _same(a, b), f"output {i} differs under PDL in {_wrong(a, b)} elements"
    _check_allreduce(res[0][:2], D.view(S, H))


@pytest.fixture(params=DTYPES, ids=DT_IDS)
def dt(request):
    return request.param


def _consumers(dt, dev, x, x32):
    """name -> consumer factory.  x(n) is a view of the first n elements of the producer's storage-type output, x32(n)
    of its fp32 output; everything else is made here, before the launch pair."""
    from videollama2_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(3)
    rnd = lambda *shape, s=1.0: (torch.randn(shape, generator=g) * s).to(dt).to(dev)
    small = lambda *shape: torch.randint(-2, 3, shape, generator=g).to(dt).to(dev)
    gamma, beta = rnd(512, s=0.1) + 1, rnd(512, s=0.1)
    inv = (1.0 / (1e4 ** (torch.arange(0, 64, 2, dtype=torch.float32) / 64))).to(dev)
    Hq, Hkv, D = 4, 2, 64
    width = (Hq + 2 * Hkv) * D
    c = {}

    def simple(fn):
        return lambda: fn

    c["layernorm"] = simple(lambda: [ops.layernorm(x(64 * 512).view(64, 512), gamma, beta, 1e-5)])
    c["layernorm_residual_act"] = simple(lambda: [ops.layernorm(x(64 * 512).view(64, 512), gamma, beta, 1e-5,
                                                                act=ops.ACT_SILU,
                                                                residual=x(2 * 64 * 512)[64 * 512:].view(64, 512))])
    rnd_wide = (rnd(8192, s=0.1) + 1, rnd(8192, s=0.1))
    c["layernorm_wide"] = simple(lambda: [ops.layernorm(x(8 * 8192).view(8, 8192), rnd_wide[0], rnd_wide[1], 1e-5)])
    c["rmsnorm"] = simple(lambda: [ops.rmsnorm(x(64 * 512).view(64, 512), gamma, 1e-5)])
    c["rmsnorm_wide"] = simple(lambda: [ops.rmsnorm(x(8 * 8192).view(8, 8192), rnd_wide[0], 1e-5)])
    c["row_sumsq"] = simple(lambda: [ops.row_sumsq(x(64 * 512).view(64, 512))])
    c["row_stats"] = simple(lambda: list(ops.row_stats(x(64 * 512).view(64, 512))))
    w_gemv = small(1024, 4096)
    c["gemv"] = simple(lambda: [ops.gemv(x(4096), w_gemv, rms_eps=1e-5)])
    c["gemv_swiglu"] = simple(lambda: [ops.gemv(x(4096), w_gemv, act=ops.ACT_SWIGLU)])
    w_sk = small(512, 1024)
    c["gemm_skinny"] = simple(lambda: [ops.gemm_skinny(x(8 * 1024).view(8, 1024), w_sk)])
    w_gg = small(256, 512)
    c["gemm"] = simple(lambda: [ops.gemm(x(128 * 512).view(128, 512), w_gg)])

    def attention():
        qkv = x(64 * width).view(64, width)
        return [ops.attention(qkv[:, :Hq * D], qkv[:, Hq * D:(Hq + Hkv) * D], qkv[:, (Hq + Hkv) * D:], B=1, S=64, Hq=Hq,
                              Hkv=Hkv, D=D, causal=True, scale=D ** -0.5)]
    c["attention"] = simple(attention)
    n_pos = 48

    def attention_decode():
        cache = x(n_pos * width).view(n_pos, width)
        q = x(n_pos * width + Hq * D)[n_pos * width:]
        return [ops.attention_decode(q, cache[:, Hq * D:(Hq + Hkv) * D], cache[:, (Hq + Hkv) * D:], n_pos=n_pos, Hq=Hq,
                                     Hkv=Hkv, D=D, scale=D ** -0.5)]
    c["attention_decode"] = simple(attention_decode)
    pos_dev = torch.tensor([n_pos - 1], device=dev, dtype=torch.int32)
    ws = ops.decode_workspace(dev, Hq, Hkv, D)

    def attention_decode_dyn():
        cache = x(n_pos * width).view(n_pos, width)
        q = x(n_pos * width + Hq * D)[n_pos * width:]
        out = torch.empty((1, Hq * D), device=dev, dtype=dt)
        return [ops.attention_decode_dyn(q, cache[:, Hq * D:(Hq + Hkv) * D], cache[:, (Hq + Hkv) * D:], pos_dev, Hq=Hq,
                                         Hkv=Hkv, D=D, scale=D ** -0.5, out=out, workspace=ws)]
    c["attention_decode_dyn"] = simple(attention_decode_dyn)

    def rope():                                        # in place on the producer's output
        qkv = x(16 * width).view(16, width)
        ops.rope_inplace(qkv, 16, Hq, Hkv, D, 0, Hq * D, 5, inv)
        return [qkv]
    c["rope_inplace"] = simple(rope)

    def rope_append():
        cache = torch.zeros((8, width), device=dev, dtype=dt)
        pos = torch.tensor([3], device=dev, dtype=torch.int32)

        def run():
            row = x(width).view(1, width)
            ops.decode_rope_append(row, cache, pos, Hq, Hkv, D, inv, interleaved=True)
            return [cache, row]
        return run
    c["decode_rope_append"] = rope_append
    ids = torch.tensor([5, 0, -3, 63, 17], device=dev, dtype=torch.int64)
    dst = torch.tensor([0, 1, 2, 5, 6], device=dev, dtype=torch.int32)

    def splice():
        out = torch.zeros((8, 512), device=dev, dtype=dt)

        def run():
            return [ops.embed_splice(ids, dst, x(64 * 512).view(64, 512), out)]
        return run
    c["embed_splice"] = splice
    w9c, g64, b64 = rnd(9, 64, s=0.3), rnd(64, s=0.1) + 1, rnd(64, s=0.1)
    c["dwconv3x3_ln_silu"] = simple(lambda: list(ops.dwconv3x3_ln_silu(x(2 * 8 * 8 * 64).view(2, 8, 8, 64), w9c, g64,
                                                                      b64, 1e-5)))
    s_se = torch.rand((2, 64), generator=g).to(dev)

    def se():                                          # in place on the producer's output
        y = x(2 * 8 * 8 * 64).view(2, 8, 8, 64)
        ops.se_scale(y, s_se)
        return [y]
    c["se_scale"] = simple(se)
    c["patch_im2col"] = simple(lambda: [ops.patch_im2col(x(2 * 3 * 28 * 28).view(2, 3, 28, 28), 14, 640)])
    c["conv3d_im2col"] = simple(lambda: [ops.conv3d_im2col(x(2 * 4 * 4 * 64).view(2, 4, 4, 64), 1)])
    wpe, pos_pe, cls_pe = rnd(64, 640, s=0.05), rnd(5, 64), rnd(64)
    wpe[:, 588:] = 0
    c["patch_embed"] = simple(lambda: [ops.patch_embed(x(2 * 3 * 28 * 28).view(2, 3, 28, 28), wpe, pos_pe, 14, cls=cls_pe,
                                                       gamma=g64, beta=b64)])
    c["clip_embed_finish"] = simple(lambda: [ops.clip_embed_finish(x(2 * 4 * 64).view(8, 64), cls_pe, pos_pe, g64, b64, 2,
                                                                   1e-5)])
    return c


F32_CONSUMERS = ["sample_token", "process_logits"]
INPLACE = {"rope_inplace", "decode_rope_append", "se_scale", "process_logits"}


def _f32_consumers(dt, dev, x32):
    from videollama2_b200 import ops
    V = 32000
    params = ops.sampling_params(1.0, 50, 0.9, 1234, dev)
    counter = torch.zeros((1,), device=dev, dtype=torch.int64)
    pparams = ops.logits_process_params(V, dev, repetition_penalty=1.3, no_repeat_ngram_size=2, min_new_tokens=2,
                                        eos_token_ids=[2], bad_words_ids=[[7, 9]], suppress_tokens=[11, 12])
    history = torch.tensor([3, 7, 5, 3, 7], device=dev, dtype=torch.int64)
    n_dev = torch.tensor([4], device=dev, dtype=torch.int64)

    def sample():
        out = torch.full((1,), -1, device=dev, dtype=torch.int64)

        def run():
            return [ops.sample_token(x32(V), params, counter, 3, out, dt)]
        return run

    def process():                                     # in place on the producer's fp32 output
        def run():
            return [ops.process_logits(x32(V), pparams, history, n_dev, 1, dt)]
        return run
    return {"sample_token": sample, "process_logits": process}


CONSUMERS = ["layernorm", "layernorm_residual_act", "layernorm_wide", "rmsnorm", "rmsnorm_wide", "row_sumsq", "row_stats",
             "gemv", "gemv_swiglu", "gemm_skinny", "gemm", "attention", "attention_decode", "attention_decode_dyn",
             "rope_inplace", "decode_rope_append", "embed_splice", "dwconv3x3_ln_silu", "se_scale", "patch_im2col",
             "conv3d_im2col", "patch_embed", "clip_embed_finish"]


def test_every_consumer_reads_after_the_producer(slow, cuda):
    """Every other entry point behind the slow GEMM: the same bits with PDL on as off."""
    x = lambda n: slow.out.view(-1)[:n]
    x32 = lambda n: slow.out32.view(-1)[:n]
    cons = _consumers(slow.dt, cuda, x, x32)
    assert sorted(cons) == sorted(CONSUMERS)
    for name in CONSUMERS:
        check_raw(slow, cons[name], what=name, inplace=name in INPLACE)
    f32 = _f32_consumers(slow.dt, cuda, x32)
    for name in F32_CONSUMERS:
        check_raw(slow, f32[name], f32=True, what=name, inplace=name in INPLACE)


# ---------------------------------------------------------------------------------------------------------------------
# b. write after read
# ---------------------------------------------------------------------------------------------------------------------
def check_war(slow, consumer, what):
    (_, c_off), (_, c_on) = run_pair(slow, consumer)
    assert _same(c_off, slow.D), f"{what}: C differs from D with PDL off"
    assert _same(c_on, slow.D), \
        f"{what}: wrote into the producer's A before the producer finished reading it ({_wrong(c_on, slow.D)} of " \
        f"{c_on.numel()} elements of C wrong)"


def test_preprocess_does_not_overwrite_the_producers_input(slow, cuda):
    """vl2_preprocess_frames' tmp is the last 5376 bytes of the GEMM's A."""
    frames = torch.from_numpy(np.random.default_rng(4).integers(0, 256, (1, 40, 64, 3), dtype=np.uint8)).to(cuda)

    def consumer():
        a, keep = _preprocess_args(slow.dt, cuda, frames, tmp=slow.tail(64 * 28 * 3))

        def run():
            _abi(slow.dt, "vl2_preprocess_frames", C.byref(a))
            return [keep["u8"]]
        return run
    check_war(slow, consumer, "vl2_preprocess_frames")


def test_waiting_kernels_do_not_overwrite_the_producers_input(slow, cuda):
    """Controls: kernels that wait, writing into the GEMM's A tail."""
    from videollama2_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(5)
    xin = (torch.randn((8, 512), generator=g) + 3).to(slow.dt).to(cuda)
    gamma = torch.ones((512,), device=cuda, dtype=slow.dt)
    beta = torch.ones((512,), device=cuda, dtype=slow.dt)
    nb = 8 * 512 * xin.element_size()
    tail = lambda: slow.tail(nb).view(slow.dt).view(8, 512)

    def ln():
        return lambda: [ops.layernorm(xin, gamma, beta, 1e-5, out=tail())]

    def rms():
        return lambda: [ops.rmsnorm(xin, gamma, 1e-5, out=tail())]

    def gemm():
        w = torch.ones((512, 512), device=cuda, dtype=slow.dt)
        return lambda: [ops.gemm(xin, w, out=tail())]
    for name, cons in (("layernorm", ln), ("rmsnorm", rms), ("gemm", gemm)):
        check_war(slow, cons, name)


# ---------------------------------------------------------------------------------------------------------------------
# c. the engine
# ---------------------------------------------------------------------------------------------------------------------
GEN_CFGS = [("tiny", torch.bfloat16), ("tiny_qwen2", torch.bfloat16), ("tiny", torch.float16)]


@pytest.fixture(scope="module", params=GEN_CFGS, ids=["tiny", "tiny_qwen2", "tiny-fp16"])
def gen(request, cuda):
    from oracle import synth
    from helpers import engine_config
    from videollama2_b200.model import VLLMs
    name, dt = request.param
    cfg = synth.CONFIGS[name]
    sd = synth.state_dict(cfg)
    px, ids = synth.inputs(cfg)
    if dt == torch.bfloat16:
        model = build_engine(cfg, sd, cuda)
    else:
        ec = engine_config(cfg)
        model = VLLMs[ec.model_type].from_state_dict(ec, sd, device=cuda, dtype=dt)
    return model, ids, [(px.to(cuda).to(dt), "video")]


def _cudart():
    """The CUDA runtime torch loaded (the graph handles it returns belong to it)."""
    torch.cuda.init()
    with open("/proc/self/maps") as fh:
        paths = sorted({m.group(0) for m in re.finditer(r"/\S*libcudart\.so[.\d]*", fh.read())})
    lib = C.CDLL(paths[0] if paths else "libcudart.so.12")
    return lib


class _EdgeData(C.Structure):      # cudaGraphEdgeData
    _fields_ = [("from_port", C.c_ubyte), ("to_port", C.c_ubyte), ("type", C.c_ubyte), ("reserved", C.c_ubyte * 5)]


PROGRAMMATIC = 1                   # cudaGraphDependencyTypeProgrammatic


def graph_edges(graph):
    """{(edge type, from port): count} of the captured graph (cudaGraphGetEdges_v2)."""
    rt = _cudart()
    fn = rt.cudaGraphGetEdges_v2
    fn.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_size_t)]
    fn.restype = C.c_int
    h = C.c_void_p(graph.raw_cuda_graph())
    n = C.c_size_t(0)
    assert fn(h, None, None, None, C.byref(n)) == 0
    frm, to, data = (C.c_void_p * n.value)(), (C.c_void_p * n.value)(), (_EdgeData * n.value)()
    assert fn(h, frm, to, data, C.byref(n)) == 0
    hist = {}
    for e in data[:n.value]:
        hist[(e.type, e.from_port)] = hist.get((e.type, e.from_port), 0) + 1
    return hist


def programmatic(hist):
    return sum(v for (t, _), v in hist.items() if t == PROGRAMMATIC)


@pytest.fixture
def kept_graphs(monkeypatch):
    """torch.cuda.CUDAGraph objects keep their cudaGraph_t (so that raw_cuda_graph() can be read after capture)."""
    orig = torch.cuda.CUDAGraph
    monkeypatch.setattr(torch.cuda, "CUDAGraph", lambda *a, **k: orig(keep_graph=True))


PROC = dict(repetition_penalty=1.3, no_repeat_ngram_size=2)
SAMPLED = dict(do_sample=True, temperature=1.5, top_p=0.95, top_k=50)


def test_decode_graphs_with_pdl_match_and_have_programmatic_edges(gen, cuda, kept_graphs):
    """Same ids and last logits with decode_pdl on as off, and proof that the mode was exercised: the captured graphs
    have programmatic edges with it and none without.  Measured on an H100 80GB HBM3: the tiny configurations' decode
    graphs have 15 (greedy) or 16 (sampled, processed) edges of type cudaGraphDependencyTypeProgrammatic, all from port
    cudaGraphKernelNodePortProgrammatic, and 3 to 5 full-dependency edges around the torch kernels."""
    model, ids, imgs = gen
    dec = model.get_model().decoder
    kinds = {"greedy": (dict(do_sample=False), "_decode_graph"),
             "sampled": (SAMPLED, "_decode_graph_sampled"),
             "processed": ({**PROC, "do_sample": False}, "_decode_graph_processed")}
    res = {}
    saved = dec.decode_pdl
    model.enable_cuda_graphs(True)
    try:
        for pdl in (False, True):
            dec.decode_pdl = pdl
            dec._drop_decode_graphs()
            for kind, (kw, attr) in kinds.items():
                g = torch.Generator(device=cuda).manual_seed(7)
                toks = model.generate(ids, images=imgs, max_new_tokens=8, eos_token_id=None, generator=g, **kw)
                graph = getattr(dec, attr)
                assert graph is not None, kind
                hist = graph_edges(graph[0])
                print(f"{kind} decode graph, decode_pdl={pdl}: edges (type, from port) -> count {hist}")
                res[(pdl, kind)] = (toks.clone(), dec.decode_graph_logits.clone(), programmatic(hist))
    finally:
        dec.decode_pdl = saved
        model.enable_cuda_graphs(False)
    for kind in kinds:
        (t0, l0, e0), (t1, l1, e1) = res[(False, kind)], res[(True, kind)]
        assert torch.equal(t0, t1), kind
        assert _same(l0, l1), f"{kind}: last logits differ in {_wrong(l0, l1)} elements"
        assert e0 == 0, f"{kind}: programmatic edges without decode_pdl"
        assert e1 > 0, f"{kind}: no programmatic edge in the decode graph with decode_pdl"


def test_eager_paths_under_pdl(gen, cuda):
    """encode_images_or_videos, prefill (all logits, with cache) and the device preprocessing, eager, PDL on == off."""
    from videollama2_b200 import ops, preprocess as pp
    from oracle import preprocess_ref as P
    model, ids, imgs = gen
    dec = model.get_model().decoder
    assert getattr(model, "_vision_cache", None) is None
    frames = torch.from_numpy(np.random.default_rng(6).integers(0, 256, (3, 45, 80, 3), dtype=np.uint8)).to(cuda)

    def flat(o):
        if isinstance(o, torch.Tensor):
            return [o.clone()]
        if isinstance(o, (list, tuple)):
            return [t for x in o for t in flat(x)]
        return []
    res = []
    for on in (False, True):
        with ops.pdl(on):
            enc = flat(model.encode_images_or_videos(imgs))
            _, _, _, emb, _ = model.prepare_inputs_labels_for_multimodal(ids, None, None, None, imgs)
            x = emb[0].to(dec.dtype).contiguous()
            logits, hidden = dec.prefill(x, all_logits=True, keep_cache=True)
            px, u8 = pp.preprocess_frames(frames, 28, P.CLIP_MEAN, P.CLIP_STD, return_u8=True, dtype=dec.dtype)
            torch.cuda.synchronize()
        res.append(enc + [logits.clone(), hidden.clone(), dec.kv[0][:x.shape[0]].clone(), px.clone(), u8.clone()])
    assert len(res[0]) == len(res[1]) and len(res[0]) > 5
    for i, (a, b) in enumerate(zip(res[1], res[0])):
        assert _same(a, b), f"tensor {i} differs under PDL in {_wrong(a, b)} of {a.numel()} elements"


def test_nested_pdl_blocks_keep_the_outer_mode(gen, cuda):
    """A graph captured in an ops.pdl(True) block after an inner ops.pdl(False) block has closed still has programmatic
    edges (the inner block restores the outer mode), and one captured after the outer block has none (VL2_PDL unset)."""
    from videollama2_b200 import ops
    model, _, _ = gen
    dec = model.get_model().decoder
    if os.environ.get("VL2_PDL") == "1":
        pytest.skip("VL2_PDL=1 turns PDL on outside every block")
    x = torch.randn((4, dec.H), generator=torch.Generator().manual_seed(8)).to(dec.dtype).to(cuda)
    gamma = torch.ones((dec.H,), device=cuda, dtype=dec.dtype)

    def capture():
        ops.rmsnorm(ops.rmsnorm(x, gamma, 1e-5), gamma, 1e-5)      # warm-up outside the capture
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph(keep_graph=True)
        with torch.cuda.graph(g):
            y = ops.rmsnorm(x, gamma, 1e-5)
            ops.rmsnorm(y, gamma, 1e-5)
            ops.rmsnorm(y, gamma, 1e-5)
        return programmatic(graph_edges(g))
    with ops.pdl(True):
        with ops.pdl(False):
            assert capture() == 0
        assert capture() > 0
    assert capture() == 0
