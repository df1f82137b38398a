"""The tensor-parallel all-reduce (vl2_tp_allreduce_stats) at world sizes 1-8, and the TP-8 decoder shards of config 5
(Qwen2-72B over 8 GPUs), on ONE GPU, bit for bit.

The kernel takes every rank's buffers as plain device pointers, so the ranks here are separate allocations on one device,
launched one after another in stream order.  Its barriers only wait until a signal-pad word reaches `epoch`; before
every launch `launch_rank` raises every word the launch will wait on to epoch + 1000 and asserts on the host that it did,
so no launch can spin (and none can reach the kernel's spin-limit trap).  No test relies on two kernels running at once.

1. The kernel on both builds, W in {1, 2, 3, 4, 5, 7, 8} x S in {1, W - 1, 7W + 3, 1776, 2 SMs W + 5} x H in {8, 2056,
   3584, 8192}, buffers taller than S filled with a NaN whose payload no arithmetic produces ("not written"):
   * ownership: after rank r's launch exactly rows [r ceil(S/W), min(S, (r + 1) ceil(S/W))) have been added to every
     rank's xout and stats; rows >= S and the partials never change;
   * sum: every rank's xout is the fp32 sum of the partials in rank order, rounded once (`expected_sum`), on rows whose
     fp32 sum depends on the order and on fp16's overflow, subnormal and inf - inf rows;
   * statistics: the sum of squares of the ROUNDED outputs, within (8 ceil(H / 2048) + 8) 2^-24 of the fp64 value
     (each thread's fma chain plus the block tree), exactly on integer rows, inf on rows holding inf;
   * protocol: a launch of rank r raises pads[s][r] and pads[s][8 + r] by one for every s < W and leaves its block
     counter (word 16) at 0, so a second launch without re-arming signals again.
2. Config 5's shard geometry (per rank H 8192, Hq 8, Hkv 1, D 128, I 3696; the QKV shard's RoPE ends at column 1152,
   inside a tile) through the real shard_state_dict and repacking, against the unsharded engine: the column-parallel
   GEMMs equal the unsharded columns bit for bit, the row-parallel GEMMs reduced by the kernel equal the unsharded GEMM
   on integer data, and eight threads running TPDecoderEngine._layer with the kernel as their all-reduce agree bit for
   bit and match the fp32 oracle."""
import ctypes as C
import math
import threading

import numpy as np
import pytest
import torch

DTYPES = [torch.bfloat16, torch.float16]
DT_IDS = ["bf16", "fp16"]
WORLDS = [1, 2, 3, 4, 5, 7, 8]
WIDTHS = [8, 2056, 3584, 8192]
MARK16 = 0x7FA5          # a NaN of the storage type that no conversion produces: "not written"
MARK32 = 0x7FA5A5A5      # the same for the fp32 statistics
GUARD = 3                # rows past S in every buffer
F32_U = 2.0 ** -24


# ---------------------------------------------------------------------------------------------------------------------
# host-side expectation (numpy; test_exact_checker.py shows on the CPU that it tells the right answer from near misses)
# ---------------------------------------------------------------------------------------------------------------------
def to_storage(x32: np.ndarray, dt) -> np.ndarray:
    """fp32 -> storage type dt, round to nearest even (fp16: subnormals kept, +-inf from 65520 on), as fp32 values."""
    x32 = np.asarray(x32, np.float32)
    if dt == torch.float16:
        with np.errstate(over="ignore"):
            return x32.astype(np.float16).astype(np.float32)
    u = x32.view(np.uint32)
    r = (((u + np.uint32(0x7FFF) + ((u >> 16) & 1)) >> 16) << 16).view(np.float32)   # wraps only on negative NaNs
    return np.where(np.isnan(x32), np.float32(np.nan), r)


def expected_sum(parts: np.ndarray, dt) -> np.ndarray:
    """The all-reduce of parts [W, S, H] (fp32 holding storage-type values): fp32 sum in rank order starting from +0,
    rounded once to dt."""
    acc = np.zeros(parts.shape[1:], np.float32)
    with np.errstate(over="ignore", invalid="ignore"):
        for p in parts:
            acc += p
    return to_storage(acc, dt)


def stats_violations(stats: np.ndarray, x: np.ndarray) -> np.ndarray:
    """Rows whose statistic is not the sum of squares of the rounded outputs x [S, H]: within (8 ceil(H / 2048) + 8)
    2^-24 of the fp64 value (each of 256 threads chains ceil(H / 2048) x 8 fmas, the block sum adds 8 levels), equal
    on integer rows with a sum below 2^24, inf on rows holding inf, NaN on rows holding NaN."""
    x64 = x.astype(np.float64)
    with np.errstate(over="ignore", invalid="ignore"):
        ss = (x64 * x64).sum(1)
        got = stats.astype(np.float64)
        tol = (8 * math.ceil(x.shape[1] / 2048) + 8) * F32_U * ss
        exact = np.all(np.isfinite(x64) & (x64 == np.round(x64)), 1) & (ss < 2.0 ** 24)
        ok = np.where(exact, got == ss, np.abs(got - ss) <= tol)
        ok |= np.isinf(ss) & (got == ss)
        ok |= np.isnan(ss) & np.isnan(got)
    return np.nonzero(~ok)[0]


PROBE = {torch.bfloat16: (2.0 ** 24, 1.0), torch.float16: (65504.0, 2.0 ** -24)}   # (big, tiny): big + tiny == big in fp32


def make_partials(W: int, S: int, H: int, dt, seed: int) -> np.ndarray:
    """Partials [W, S, H] (fp32 holding dt values).  Rows cycle through four kinds:
      0: N(0, 1); W >= 3: column 0 is [big, tiny, -big] (fp32 in rank order: 0; exact: tiny; bf16 reversed: tiny),
         column 1 [big, -big, tiny] (in rank order: tiny; fp16 reversed: 0), later ranks 0 there;
      1: integers in [-4, 4] (exact sum and statistic);
      2: N(0, 1) with +inf in rank 0's column 1; fp16 and W >= 2 also: 65504 + 15.984375 (-> 65504), 65504 + 16
         (-> inf), -65504 - 16 (-> -inf), 2^-14 - (2^-14 - 2^-24) (-> 2^-24), -5 2^-24 + 2 2^-24 (subnormal);
      3: N(0, 1); W >= 2: column 0 is inf + (-inf) (-> NaN)."""
    rng = np.random.default_rng(seed)
    p = to_storage(rng.standard_normal((W, S, H), dtype=np.float32), dt)
    p[:, 1::4] = rng.integers(-4, 5, p[:, 1::4].shape).astype(np.float32)
    big, tiny = PROBE[dt]
    if W >= 3:
        p[:, 0::4, :2] = 0
        p[:3, 0::4, 0] = np.array([big, tiny, -big], np.float32)[:, None]
        p[:3, 0::4, 1] = np.array([big, -big, tiny], np.float32)[:, None]
    p[0, 2::4, 1] = np.inf
    if dt == torch.float16 and W >= 2:
        p[:, 2::4, 2:7] = 0
        rows = np.array([[65504.0, 15.984375], [65504.0, 16.0], [-65504.0, -16.0], [2.0 ** -14, -(2.0 ** -14 - 2.0 ** -24)],
                         [-5 * 2.0 ** -24, 2 * 2.0 ** -24]], np.float32).T
        p[:2, 2::4, 2:7] = rows[:, None, :]
    if W >= 2:
        p[:, 3::4, 0] = 0
        p[0, 3::4, 0], p[1, 3::4, 0] = np.inf, -np.inf
    return p


# ---------------------------------------------------------------------------------------------------------------------
# one rank's launch
# ---------------------------------------------------------------------------------------------------------------------
def _marked(shape, dev, dt):
    mark, bits = (MARK32, torch.int32) if dt == torch.float32 else (MARK16, torch.int16)
    return torch.full(shape, mark, device=dev, dtype=bits).view(dt)


def _written(t: torch.Tensor) -> torch.Tensor:
    if t.dtype == torch.float32:
        return t.view(torch.int32) != MARK32
    return t.view(torch.int16) != MARK16


def make_buffers(W: int, S: int, H: int, dt, dev) -> dict:
    """Every rank's partial, xout and stats, GUARD rows taller than S and marked "not written", and zeroed pads."""
    return {"part": [_marked((S + GUARD, H), dev, dt) for _ in range(W)],
            "xout": [_marked((S + GUARD, H), dev, dt) for _ in range(W)],
            "stats": [_marked((S + GUARD,), dev, torch.float32) for _ in range(W)],
            "pads": torch.zeros((W, 32), device=dev, dtype=torch.int32)}


def assert_never_waits(pads: np.ndarray, r: int, W: int, epoch: int) -> None:
    """Every pad word rank r's launch waits on (its own words 0..W-1 and 8..8+W-1) already holds >= epoch, counting
    the one increment the launch itself makes to words r and 8 + r before it waits on them."""
    own = pads[r].astype(np.int64)
    for t in range(W):
        for w in (t, 8 + t):
            assert own[w] + (t == r) >= epoch, f"rank {r} would wait on pad word {w} ({own[w]} < epoch {epoch})"


def launch_rank(dt, bufs: dict, r: int, S: int, H: int, epoch: int, arm: bool = True) -> np.ndarray:
    """Launch rank r of W = len(bufs['part']).  `arm`: first set words 0-15 of every rank's pad to epoch + 1000 and word
    16 of rank r's to 0.  Returns the pads as they were at the launch (uint32 [W, 32])."""
    from videollama2_b200 import _lib
    W, pads = len(bufs["part"]), bufs["pads"]
    if arm:
        pads[:, :16] = epoch + 1000
        pads[r, 16] = 0
    before = pads.cpu().numpy().view(np.uint32).copy()
    assert_never_waits(before, r, W, epoch)
    a = _lib.TpAllReduceArgs(rank=r, world=W, S=S, H=H, epoch=epoch, inswitch_reduce=0)
    for s in range(W):
        a.part[s], a.xout[s] = bufs["part"][s].data_ptr(), bufs["xout"][s].data_ptr()
        a.stats[s], a.pads[s] = bufs["stats"][s].data_ptr(), pads[s].data_ptr()
    lib = _lib.load(dt)
    _lib.check(lib.vl2_tp_allreduce_stats(C.byref(a), torch.cuda.current_stream().cuda_stream), "vl2_tp_allreduce_stats", lib)
    return before


def check_signalled(bufs: dict, before: np.ndarray, r: int, what: str) -> None:
    """Rank r's launch raised pads[s][r] and pads[s][8 + r] of every rank s by one and changed no other word; its
    block counter (word 16) is back to 0."""
    after = bufs["pads"].cpu().numpy().view(np.uint32)
    want = before.copy()
    want[:, r] += 1
    want[:, 8 + r] += 1
    assert after[r, 16] == 0, f"{what}: rank {r}'s block counter left at {after[r, 16]}"
    assert np.array_equal(after, want), f"{what}: pads after rank {r}'s launch\n{after[:, :17]}\nexpected\n{want[:, :17]}"


def _same(got: torch.Tensor, want: torch.Tensor) -> torch.Tensor:
    """Element-wise: the same bits, or both NaN."""
    bits = torch.int32 if got.dtype == torch.float32 else torch.int16
    return (got.view(bits) == want.view(bits)) | (torch.isnan(got) & torch.isnan(want))


def _row_spans(S: int, W: int):
    per = -(-S // W)
    return [(min(S, r * per), min(S, (r + 1) * per)) for r in range(W)]


# ---------------------------------------------------------------------------------------------------------------------
# 1. the kernel at world 1-8
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(params=DTYPES, ids=DT_IDS)
def dt(request):
    return request.param


@pytest.mark.gpu
@pytest.mark.parametrize("H", WIDTHS)
@pytest.mark.parametrize("W", WORLDS)
def test_allreduce_rows_sum_statistics_protocol(cuda, dt, W, H):
    sms = torch.cuda.get_device_properties(cuda).multi_processor_count
    sizes = sorted({s for s in (1, W - 1, 7 * W + 3, 1776, 2 * sms * W + 5) if s >= 1})
    for S in sizes:
        what = f"{DT_IDS[DTYPES.index(dt)]} W {W} S {S} H {H}"
        parts = make_partials(W, S, H, dt, seed=1000 * W + S + H)
        want = torch.from_numpy(expected_sum(parts, dt)).to(cuda).to(dt)
        bufs = make_buffers(W, S, H, dt, cuda)
        for s in range(W):
            bufs["part"][s][:S] = torch.from_numpy(parts[s]).to(cuda).to(dt)
        part0 = [p.clone() for p in bufs["part"]]
        owned = torch.zeros(S + GUARD, device=cuda, dtype=torch.bool)
        for r, (lo, hi) in enumerate(_row_spans(S, W)):
            before = launch_rank(dt, bufs, r, S, H, epoch=5 + r)
            check_signalled(bufs, before, r, what)
            owned[lo:hi] = True
            for s in range(W):
                wx, ws = _written(bufs["xout"][s]), _written(bufs["stats"][s])
                assert torch.equal(wx, owned[:, None].expand_as(wx)), \
                    f"{what}: after rank {r} (rows [{lo}, {hi})) rank {s}'s xout rows written: " \
                    f"{torch.nonzero(wx.any(1)).flatten().tolist()[:8]}..."
                assert torch.equal(ws, owned), f"{what}: after rank {r} rank {s}'s stats rows written: " \
                    f"{torch.nonzero(ws).flatten().tolist()[:8]}..."
        for s in range(W):
            assert torch.equal(bufs["part"][s].view(torch.int16), part0[s].view(torch.int16)), f"{what}: partial {s} changed"
            ok = _same(bufs["xout"][s][:S], want)
            if not bool(ok.all()):
                row, col = (int(v) for v in torch.nonzero(~ok)[0])
                raise AssertionError(f"{what}: rank {s}'s xout[{row}, {col}] = {float(bufs['xout'][s][row, col])}, "
                                     f"want {float(want[row, col])} (partials {parts[:, row, col].tolist()})")
            assert bool(_same(bufs["stats"][s], bufs["stats"][0]).all()), f"{what}: rank {s}'s stats differ from rank 0's"
        stats, x = bufs["stats"][0][:S].cpu().numpy(), want.float().cpu().numpy()
        bad = stats_violations(stats, x)
        assert bad.size == 0, f"{what}: statistics of rows {bad[:8].tolist()}: got {stats[bad[:4]].tolist()}, " \
            f"want {(x[bad[:4]].astype(np.float64) ** 2).sum(1).tolist()}"
        # a second launch of the last rank without re-arming its block counter: it still signals, same bits
        r = W - 1
        before = launch_rank(dt, bufs, r, S, H, epoch=5 + r, arm=False)
        check_signalled(bufs, before, r, what + " (second launch)")
        for s in range(W):
            assert bool(_same(bufs["xout"][s][:S], want).all()), f"{what}: second launch changed rank {s}'s xout"
        del bufs, part0, want
    torch.cuda.empty_cache()


@pytest.mark.gpu
@pytest.mark.parametrize("S", [1, 77, 128])
def test_allreduce_world1_zeroed_pad_self_signals(cuda, dt, S):
    """World 1 on a genuinely zeroed pad, epochs 1-4 (no arming): the launch's own arrivals are what its barriers wait
    for, so words 0 and 8 count the launches and word 16 is re-armed to 0 each time; the output is the partial."""
    H = 1024
    parts = make_partials(1, S, H, dt, seed=S)
    want = torch.from_numpy(expected_sum(parts, dt)).to(cuda).to(dt)
    bufs = make_buffers(1, S, H, dt, cuda)
    bufs["part"][0][:S] = torch.from_numpy(parts[0]).to(cuda).to(dt)
    for e in range(1, 5):
        before = launch_rank(dt, bufs, 0, S, H, epoch=e, arm=False)
        assert before[0, 0] == e - 1 and before[0, 8] == e - 1
        check_signalled(bufs, before, 0, f"epoch {e}")
        pad = bufs["pads"].cpu().numpy().view(np.uint32)[0]
        assert pad[0] == e and pad[8] == e and pad[16] == 0 and not pad[17:].any() and not pad[1:8].any()
        assert bool(_same(bufs["xout"][0][:S], want).all())
        assert not bool(_written(bufs["xout"][0][S:]).any()) and not bool(_written(bufs["stats"][0][S:]).any())
    assert stats_violations(bufs["stats"][0][:S].cpu().numpy(), want.float().cpu().numpy()).size == 0


# ---------------------------------------------------------------------------------------------------------------------
# 2. config 5's shards (Qwen2-72B, TP 8) against the unsharded layer, bf16
# ---------------------------------------------------------------------------------------------------------------------
TP = 8
S5 = 1776
POS0 = 37


def _sparse_ones(shape, density_inv: int, g, dev):
    """Entries -1, 0, 1 with P(+-1) = 1 / density_inv each (bf16)."""
    u = torch.randint(0, density_inv, shape, generator=g, device=dev)
    return ((u == 0).to(torch.int8) - (u == 1).to(torch.int8)).to(torch.bfloat16)


def _layer_state(cfg, dev) -> dict:
    """HF-named weights of one Qwen2-72B decoder layer (+ vocab-64 embedding / head) drawn on the device.  o_proj and
    down_proj hold sparse {-1, 0, 1} (two nonzeros in 128): the row-parallel GEMMs are then exact on integer inputs."""
    from videollama2_b200 import presets
    g = torch.Generator(device=dev).manual_seed(5)
    sd = {}
    for name, shape, kind in presets.state_dict_specs(cfg):
        if name.startswith("model.vision_tower.") or name.startswith("model.mm_projector."):
            continue
        if name.endswith(("o_proj.weight", "down_proj.weight")):
            sd[name] = _sparse_ones(shape, 128, g, dev)
            continue
        x = torch.randn(shape, generator=g, device=dev, dtype=torch.float32)
        x = x * shape[-1] ** -0.5 if kind == "w" else (1.0 + 0.1 * x if kind == "gain" else x * (0.02 if kind == "bias" else 0.05))
        sd[name] = x.to(torch.bfloat16)
    return sd


@pytest.fixture(scope="module")
def cfg5(cuda):
    """(config, state dict, unsharded DecoderEngine, the 8 TPDecoderEngines built by shard_state_dict + repacking)."""
    import torch.distributed as dist
    from videollama2_b200 import presets
    from videollama2_b200.model.decoder import DecoderEngine
    from videollama2_b200.model.tp_decoder import TPDecoderEngine
    cfg = presets.make_config(dict(presets.QWEN2_72B, num_hidden_layers=1, vocab_size=64), 16)
    sd = _layer_state(cfg, cuda)
    full = DecoderEngine(cfg).load_state_dict(sd, cuda)
    tp = []
    for r in range(TP):
        with pytest.MonkeyPatch.context() as m:           # the rank / world a process group would report
            m.setattr(dist, "get_rank", lambda group=None, r=r: r)
            m.setattr(dist, "get_world_size", lambda group=None: TP)
            eng = TPDecoderEngine(cfg)
        tp.append(eng.load_state_dict(sd, cuda))
    yield cfg, sd, full, tp
    del sd, full, tp
    torch.cuda.empty_cache()


def _qkv_columns(r: int, Hq: int, Hkv: int, D: int, dev) -> torch.Tensor:
    """Columns of the unsharded QKV output (q heads, then k heads, then v heads) that rank r's QKV shard produces."""
    hq, hkv = Hq // TP, Hkv // TP
    q = torch.arange(r * hq * D, (r + 1) * hq * D)
    k = Hq * D + torch.arange(r * hkv * D, (r + 1) * hkv * D)
    v = (Hq + Hkv) * D + torch.arange(r * hkv * D, (r + 1) * hkv * D)
    return torch.cat([q, k, v]).to(dev)


@pytest.mark.gpu
def test_tp8_shards_are_the_unsharded_weights(cfg5):
    """shard_state_dict + repacking at config 5's geometry: rank r's fused, permuted, gain-folded QKV rows and bias, its
    interleaved gate / up rows and its o_proj / down_proj columns are those of the unsharded engine, bit for bit."""
    cfg, _, full, tp = cfg5
    F = full.layers[0]
    I = cfg.intermediate_size // TP
    for r, eng in enumerate(tp):
        L = eng.layers[0]
        assert (eng.Hq, eng.Hkv, eng.D, eng.I, L["wqkv"].shape[0]) == (8, 1, 128, 3696, 1280)
        cols = _qkv_columns(r, full.Hq, full.Hkv, full.D, F["wqkv"].device)
        assert torch.equal(L["wqkv"], F["wqkv"][cols]) and torch.equal(L["bqkv"], F["bqkv"][cols])
        assert torch.equal(L["wgu"], F["wgu"][2 * r * I:2 * (r + 1) * I])
        assert torch.equal(L["wo"], F["wo"][:, r * 1024:(r + 1) * 1024])
        assert torch.equal(L["wd"], F["wd"][:, r * I:(r + 1) * I])
        assert torch.equal(eng.rope_table(POS0 + S5), full.rope_table(POS0 + S5))


@pytest.mark.gpu
@pytest.mark.parametrize("bn", [128, 160, 224, 1256])
def test_tp8_column_parallel_gemms_bit_exact(cfg5, cuda, bn):
    """Random residual stream, S = 1776 from position 37, the same forced tile width on both sides: rank r's QKV GEMM
    (bias + folded RMSNorm + RoPE over its first 1152 columns, a boundary inside a tile) equals the unsharded QKV's
    columns of its heads, and its SwiGLU GEMM the unsharded SwiGLU output's columns [3696 r, 3696 (r + 1))."""
    from videollama2_b200 import ops
    cfg, _, full, tp = cfg5
    F = full.layers[0]
    D, H, I = full.D, full.H, cfg.intermediate_size // TP
    x = (torch.randn((S5, H), generator=torch.Generator().manual_seed(11)) * 0.7).to(torch.bfloat16).to(cuda)
    ss = ops.row_sumsq(x)
    kw = dict(rms_in=ss, rms_eps=full.eps, bn=bn, splitk=False)
    qkv = ops.gemm(x, F["wqkv"], bias=F["bqkv"], rope=(full.rope_table(POS0 + S5), POS0, D, (full.Hq + full.Hkv) * D), **kw)
    h = ops.gemm(x, F["wgu"], act=ops.ACT_SWIGLU, **kw)
    for r, eng in enumerate(tp):
        L = eng.layers[0]
        nqk = (eng.Hq + eng.Hkv) * D
        assert nqk == 1152
        mine = ops.gemm(x, L["wqkv"], bias=L["bqkv"], rope=(eng.rope_table(POS0 + S5), POS0, D, nqk), **kw)
        want = qkv[:, _qkv_columns(r, full.Hq, full.Hkv, D, cuda)]
        diff = torch.nonzero(mine.view(torch.int16) != want.view(torch.int16))
        assert diff.numel() == 0, f"bn {bn} rank {r}: QKV differs in {diff.shape[0]} elements, first (row, col) " \
            f"{diff[0].tolist()}"
        mine = ops.gemm(x, L["wgu"], act=ops.ACT_SWIGLU, **kw)
        want = h[:, r * I:(r + 1) * I]
        diff = torch.nonzero(mine.view(torch.int16) != want.view(torch.int16))
        assert diff.numel() == 0, f"bn {bn} rank {r}: SwiGLU differs in {diff.shape[0]} elements, first (row, col) " \
            f"{diff[0].tolist()}"


def _assert_exact_premise(t64: torch.Tensor, what: str) -> None:
    """Integers of magnitude <= 256 (bf16-exact) with row sums of squares below 2^24 (fp32-exact in any order)."""
    assert torch.equal(t64, t64.round()) and float(t64.abs().max()) <= 256, f"{what}: not small integers"
    assert float(t64.pow(2).sum(1).max()) < 2.0 ** 24, f"{what}: a row's sum of squares reaches 2^24"


@pytest.mark.gpu
def test_tp8_row_parallel_gemms_reduce_to_the_unsharded_gemm(cfg5, cuda):
    """o_proj and down_proj shards called as TPDecoderEngine._layer calls them (residual on rank 0 only, output into the
    rank's partial buffer) on sparse {-1, 0, 1} activations, reduced by the kernel: every rank's result equals the
    unsharded ops.gemm(..., residual=x) and the fp64 result, its statistics equal the fp64 sums of squares, and the
    SwiGLU GEMM fed those statistics equals the one fed ops.row_sumsq of the result."""
    from videollama2_b200 import ops
    cfg, _, full, tp = cfg5
    F, H = full.layers[0], full.H
    g = torch.Generator(device=cuda).manual_seed(13)
    x = torch.randint(-8, 9, (S5, H), generator=g, device=cuda).to(torch.bfloat16)
    I = cfg.intermediate_size // TP
    cases = [("o_proj", "wo", _sparse_ones((S5, full.Hq * full.D), 4, g, cuda), full.Hq * full.D // TP),
             ("down_proj", "wd", _sparse_ones((S5, cfg.intermediate_size), 4, g, cuda), I)]
    for epoch, (name, key, a, k) in enumerate(cases, 1):
        want = ops.gemm(a, F[key], residual=x, splitk=False)
        ref = a.double() @ F[key].double().t() + x.double()
        _assert_exact_premise(ref, name)
        assert torch.equal(want.double(), ref), f"{name}: the unsharded GEMM is not exact"
        bufs = make_buffers(TP, S5, H, torch.bfloat16, cuda)
        for r, eng in enumerate(tp):
            res = x if eng.rank == 0 else None
            ops.gemm(a[:, r * k:(r + 1) * k].contiguous(), eng.layers[0][key], residual=res, out=bufs["part"][r][:S5])
            _assert_exact_premise(bufs["part"][r][:S5].double(), f"{name} partial {r}")
        for r in range(TP):
            launch_rank(torch.bfloat16, bufs, r, S5, H, epoch)
        for r, eng in enumerate(tp):
            got, st = bufs["xout"][r][:S5], bufs["stats"][r][:S5]
            assert torch.equal(got, want), f"{name}: rank {r}'s reduced stream differs from the unsharded GEMM"
            assert torch.equal(st.double(), ref.pow(2).sum(1)), f"{name}: rank {r}'s statistics are not exact"
            if name == "o_proj":
                L = eng.layers[0]
                h1 = ops.gemm(got, L["wgu"], act=ops.ACT_SWIGLU, rms_in=st.view(S5, 1), rms_eps=eng.eps)
                h2 = ops.gemm(got, L["wgu"], act=ops.ACT_SWIGLU, rms_in=ops.row_sumsq(got.contiguous()), rms_eps=eng.eps)
                assert torch.equal(h1, h2), f"rank {r}: SwiGLU fed the kernel's statistics differs"


@pytest.mark.gpu
def test_tp8_layer_in_eight_threads(cfg5, cuda):
    """Eight threads, one per rank, each running its TPDecoderEngine._layer (S = 1776 from position 37) with the kernel
    as the all-reduce: write the partial, meet at a barrier, pre-arm the own pad, launch the own rank's reduction, meet
    again (nobody's next GEMM overwrites a partial a peer still reduces).  All launches go to one stream.  The eight
    outputs are bit-identical and within relL2 1e-2 of the fp32 oracle."""
    from oracle import synth, torch_ref
    from videollama2_b200 import ops
    cfg, sd, full, tp = cfg5
    H = full.H
    x = (torch.randn((S5, H), generator=torch.Generator().manual_seed(17)) * 0.7).to(torch.bfloat16).to(cuda)
    part = [_marked((S5, H), cuda, torch.bfloat16) for _ in range(TP)]
    outs = [{"xout": [_marked((S5, H), cuda, torch.bfloat16) for _ in range(TP)],
             "stats": [_marked((S5,), cuda, torch.float32) for _ in range(TP)]} for _ in range(2)]
    pads = torch.zeros((TP, 32), device=cuda, dtype=torch.int32)
    barrier = threading.Barrier(TP, timeout=300)
    results, errors = [None] * TP, []
    stream = torch.cuda.Stream(device=cuda)
    stream.wait_stream(torch.cuda.current_stream())

    def reduce_stats(r, eng, calls):
        def _reduce_stats(gemm_into):
            S = eng._cur_rows
            gemm_into(part[r][:S])
            barrier.wait()
            epoch = len(calls) + 1
            out = outs[len(calls) % 2]
            calls.append(epoch)
            pads[r, :16] = epoch + 1000
            pads[r, 16] = 0
            bufs = {"part": part, "xout": out["xout"], "stats": out["stats"], "pads": pads}
            launch_rank(torch.bfloat16, bufs, r, S, H, epoch, arm=False)
            barrier.wait()
            return out["xout"][r][:S], out["stats"][r][:S].view(S, 1)
        return _reduce_stats

    def run(r, eng):
        try:
            with torch.cuda.stream(stream):
                eng._reduce_stats = reduce_stats(r, eng, [])
                results[r] = eng._layer(eng.layers[0], x, S5, POS0, None, ops.row_sumsq(x))[0]
        except BaseException as e:          # noqa: B902 - reported below; the others must not wait for this rank
            errors.append((r, e))
            barrier.abort()

    with torch.cuda.stream(stream):
        threads = [threading.Thread(target=run, args=(r, eng)) for r, eng in enumerate(tp)]
        for t in threads:
            t.start()
        for t in threads:
            t.join()
    for eng in tp:
        eng.__dict__.pop("_reduce_stats", None)
    torch.cuda.current_stream().wait_stream(stream)
    torch.cuda.synchronize()
    real = [(r, e) for r, e in errors if not isinstance(e, threading.BrokenBarrierError)]
    if errors:
        raise (real or errors)[0][1]
    for r in range(1, TP):
        assert torch.equal(results[r], results[0]), f"rank {r}'s layer output differs from rank 0's"
    l = synth.LlmCfg(kind="qwen2", hidden=H, inter=cfg.intermediate_size, layers=1, heads=cfg.num_attention_heads,
                     kv_heads=cfg.num_key_value_heads, vocab=64, eps=cfg.rms_norm_eps, theta=cfg.rope_theta)
    cos, sin = torch_ref.rope_cos_sin(S5, l.head_dim, l.theta, torch.float32, pos0=POS0)
    ref = torch_ref.decoder_layer(sd, l, 0, x.float(), cos.to(cuda), sin.to(cuda), torch.float32, sdpa=True)
    err = float((results[0].double() - ref.double()).norm() / ref.double().norm())
    print(f"TP-8 layer relL2 vs fp32 oracle: {err:.3e}")
    assert err <= 1e-2
