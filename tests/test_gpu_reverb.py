"""FIR convolutional reverb (reverb.cu) against exact known answers and f64 references.

The GEMM picks a tile width BN in {256, 224, 192, 128} per call and may split the tiles of a short tail wave along K; its
history of bf16 samples is appended to and compacted across calls. Every (BN, split) combination, the IR channel map, short
and long IRs, and the history edges are pinned here:
- known answers: sparse impulse trains whose output samples are each one exact product `a * bf16(h[k])`, compared with `==`;
- dense inputs: per row and per call, normalised max error <= 1e-5 against an f64 FFT convolution of the bf16-rounded operands.
The tests without a `gpu` mark check the reference helpers themselves and run without a device."""
import functools

import numpy as np
import pytest

from firewheel_b200 import AudioGraphConfig, ConvReverbNode, FirewheelGraphCtx, VolumeNode
from helpers import assert_bit_exact, f32, run_planar

SR = 48000
TOL = 1e-5


# ---- reference helpers ------------------------------------------------------------------------------------------------
def bf16_rne(x):
    """Round to nearest even to bfloat16, returned as float32 (the oracle's bf16_round, vectorised); NaN stays NaN."""
    u = np.ascontiguousarray(x, dtype=f32).view(np.uint32)
    nan = (u & np.uint32(0x7fffffff)) > np.uint32(0x7f800000)
    r = (u + np.uint32(0x7fff) + ((u >> np.uint32(16)) & np.uint32(1))) & np.uint32(0xffff0000)
    r = np.where(nan, (u | np.uint32(0x00400000)) & np.uint32(0xffff0000), r).astype(np.uint32)
    return r.view(f32)


def ref_conv(x_rows, h_rows):
    """f64 FFT convolution of the bf16-rounded operands, row by row, cut to the input length. x_rows [R][N] is the
    concatenation of all calls' inputs, h_rows [R][L] the IR row each input row uses."""
    import scipy.signal
    xb, hb = bf16_rne(x_rows).astype(np.float64), bf16_rne(h_rows).astype(np.float64)
    return scipy.signal.fftconvolve(xb, hb, axes=-1)[:, : xb.shape[1]]


def reverb_plan(V, C, T, L, sms):
    """The GEMM's launch shape for one call of T frames over V voices and C channels: (BN, tiles, tail_tiles, split).
    Mirrors reverb_pick_bn and the tail-split rule of launch_reverb (reverb.cu)."""
    tiles_mc = -(-V // 128) * C
    bn, best = 256, None
    for cand in (256, 224, 192, 128):
        waves = -(-(-(-T // cand) * tiles_mc) // sms)
        cost = waves * (max(4 * cand, 256 + 3 * cand) + 8)
        if best is None or cost < best:
            bn, best = cand, cost
    num_kb = ((L - 1 + 7) // 8 * 8 + bn + 63) // 64
    tiles = -(-T // bn) * tiles_mc
    if tiles > sms and tiles % sms:
        split = min(sms // (tiles % sms), num_kb // 16)
        if split >= 2:
            return bn, tiles, tiles % sms, split
    return bn, tiles, 0, 1


@functools.lru_cache(maxsize=None)
def shape_matrix(sms, L=4100):
    """For each (BN, split) one shape (V, C, T, L), chosen from a candidate grid: more than one voice tile and more than one time
    tile where possible, a ragged last time tile, then the least work. BN = 128 with a split needs more voice tiles than SMs in
    one call: its candidate has sms // 2 + 1 voice tiles of two channels, which at 132 SMs is V = 8449 and about 4.6 GB of
    history; every other chosen shape stays under 300 MB."""
    cands = [(V, C, T, L) for V in (1, 129, 257, 513, 771, 1030) for C in (1, 2) for T in range(8, 16385, 8)]
    cands.append((128 * (sms // 2) + 1, 2, 128, 2048))
    best = {}
    for V, C, T, Lc in cands:
        bn, _, _, split = reverb_plan(V, C, T, Lc, sms)
        key = (bn, split > 1)
        rank = (V <= 128, T <= bn, T % bn == 0, V * C * T)
        if key not in best or rank < best[key][0]:
            best[key] = (rank, (V, C, T, Lc))
    return {k: v[1] for k, v in best.items()}


KEYS = [(bn, sp) for bn in (128, 192, 224, 256) for sp in (False, True)]


def reverb_ir(L, ch, seed):
    rng = np.random.default_rng(seed)
    h = rng.standard_normal((ch, L)) * np.exp(-6.9 * np.arange(L) / L)
    h /= np.sqrt((h ** 2).sum(axis=1, keepdims=True))
    return h.astype(f32)


def impulses(V, C, lens, L, marks, seed=0):
    """Sparse impulse trains over a stream of calls of `lens` frames: x [V][C][sum(lens)] and, per row v * C + c, a list of
    (position, amplitude). Positions are drawn from `marks` (frames of interest) starting at a different mark for every row,
    plus random fill, at least L apart; amplitudes are +-2^e with e and the sign depending on the row."""
    N = int(sum(lens))
    marks = sorted({int(m) for m in marks if 0 <= m < N})
    rng = np.random.default_rng(seed)
    x = np.zeros((V * C, N), f32)
    rows = []
    for r in range(V * C):
        amp = (-1.0 if (r // 61) % 2 else 1.0) * 2.0 ** ((r % 61) - 30)
        order = marks[(r * 7) % len(marks):] + marks[:(r * 7) % len(marks)] if marks else []
        order += list(rng.integers(0, N, 4))
        pos = []
        for p in order:
            if all(abs(p - q) >= L for q in pos):
                pos.append(int(p))
        for p in pos:
            x[r, p] = amp
        rows.append([(p, amp) for p in pos])
    return x.reshape(V, C, N), rows


def impulse_answer(rows, V, C, N, h, L):
    """The exact output of an impulse train: every sample is one product a * bf16(h[c % ir_ch][k]), or zero."""
    hb = bf16_rne(h).astype(np.float64)
    y = np.zeros((V * C, N), np.float64)
    for r, imp in enumerate(rows):
        hr = hb[(r % C) % hb.shape[0]]
        for p, a in imp:
            n = min(L, N - p)
            y[r, p:p + n] = a * hr[:n]
    return y.astype(f32).reshape(V, C, N)


def assert_equal_samples(got, want, what):
    bad = np.argwhere(got != want)
    if len(bad):
        i = tuple(bad[0])
        raise AssertionError(f"{what}: {len(bad)} of {got.size} samples differ; first at (voice, channel, frame) {i}: got {got[i]!r} want {want[i]!r}")


def assert_close_per_row(y, ref, lens, what, zero_rows=()):
    """Normalised max error <= TOL for every row and every call; rows zero so far must give exact zeros."""
    t0 = 0
    for k, T in enumerate(lens):
        for r in range(y.shape[0]):
            g, w = y[r, t0:t0 + T].astype(np.float64), ref[r, t0:t0 + T]
            m = np.max(np.abs(w)) if T else 0.0
            if m == 0.0:
                assert np.all(g == 0), f"{what}: row {r} call {k}: a silent row gave non-zero output {g[g != 0][:4]}"
                continue
            e = float(np.max(np.abs(g - w)) / m)
            assert e <= TOL, f"{what}: row {r} call {k} (frames {t0}..{t0 + T}): normalised max error {e:.3g}"
        t0 += T
    for r in zero_rows:
        assert np.all(y[r] == 0), f"{what}: zero input row {r} gave non-zero output"


# ---- running the product ----------------------------------------------------------------------------------------------
def reverb_ctx(lib, C, ir, V, F=256, max_call_frames=0):
    """graph_in -> ConvReverb(ir) -> graph_out with C channels: one fused-chain stage for C <= 2, the generic lowering (one
    launch per channel) above that."""
    cx = FirewheelGraphCtx(lib, AudioGraphConfig(num_graph_inputs=C, num_graph_outputs=C, num_voices=V, max_call_frames=max_call_frames))
    g = cx.graph
    rv = g.add_node(C, C, ConvReverbNode(ir))
    for c in range(C):
        g.connect(g.graph_in_node(), c, rv, c, False)
        g.connect(rv, c, g.graph_out_node(), c, False)
    proc = cx.activate(SR, C, C, F)
    st = cx.update()
    assert st.graph_error is None, cx.last_error()
    return cx, proc, rv


def close(cx, proc):
    proc.free(); cx.update(); cx.free()


def stream(lib, C, ir, x, lens, F=256, max_call_frames=0):
    """x [V][C][sum(lens)] sent as consecutive calls of `lens` frames through one context; returns y [V][C][sum(lens)] and the masks."""
    cx, proc, _ = reverb_ctx(lib, C, ir, x.shape[0], F, max_call_frames)
    ys, masks, t0 = [], [], 0
    for T in lens:
        y, m = run_planar(proc, np.ascontiguousarray(x[:, :, t0:t0 + T]), C)
        ys.append(y); masks.append(m); t0 += T
    close(cx, proc)
    return np.concatenate(ys, axis=2), masks


def call_marks(lens, bn):
    """Frames where a kernel boundary lies: call starts and ends, BN-wide time-tile edges inside each call."""
    marks, s = [], 0
    for T in lens:
        marks += [s, s + 1, s + T - 1]
        for j in range(1, -(-T // bn)):
            marks += [s + j * bn - 1, s + j * bn]
        s += T
    return marks


def dense(V, C, N, seed, zero_every=11):
    """Seeded uniform input, rows scaled by 2^-6 .. 2^6, every `zero_every`-th row all zero. Returns x and the zero rows."""
    rng = np.random.default_rng(seed)
    x = (rng.random((V * C, N), dtype=np.float64) * 2 - 1).astype(f32)
    x *= (2.0 ** ((np.arange(V * C) * 5) % 13 - 6)).astype(f32)[:, None]
    zero = [r for r in range(V * C) if r % zero_every == zero_every // 2]
    x[zero] = 0
    return x.reshape(V, C, N), zero


def sample_rows(V, C, n=24, seed=0):
    """Rows checked against the FFT reference: the first and last voices, both sides of the first voice tile boundary, a spread."""
    vs = {0, V - 1, min(127, V - 1), min(128, V - 1)} | set(np.random.default_rng(seed).integers(0, V, n).tolist())
    return sorted(v * C + c for v in vs for c in range(C))


def check_dense(y, x, h, lens, rows, what, zero_rows=()):
    V, C, N = x.shape
    xr, yr = x.reshape(V * C, N), y.reshape(V * C, N)
    ref = ref_conv(xr[rows], h[[(r % C) % h.shape[0] for r in rows]])
    assert_close_per_row(yr[rows], ref, lens, what)
    for r in zero_rows:
        assert np.all(yr[r] == 0), f"{what}: zero input row {r} gave non-zero output"


@pytest.fixture(scope="module")
def sms(gpu):
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


# ---- CPU: the helpers themselves --------------------------------------------------------------------------------------
def test_bf16_rne_matches_oracle(oracle):
    edge = [0x3f808000, 0x3f818000, 0x3f807fff, 0x3f808001, 0xbf808000, 0xbf818000, 0x00000000, 0x80000000, 0x7f800000, 0xff800000,
            0x7fc00000, 0xffc00000, 0x7f800001, 0xff800001, 0x7fbfffff, 0x7f7fffff, 0xff7fffff, 0x7f7f7fff, 0x7f7f8000, 0x00000001,
            0x00008000, 0x00018000, 0x007fffff, 0x807fffff, 0x00800000, 0x3f800000, 0x3f7fffff]
    rand = np.random.default_rng(1).integers(0, 1 << 32, 4000, dtype=np.uint64).astype(np.uint32).tolist()
    u = np.array(edge + rand, np.uint32)
    got = bf16_rne(u.view(f32)).view(np.uint32)
    want = np.array([np.float32(oracle.bf16_round(float(v))) for v in u.view(f32)], f32).view(np.uint32)
    nan = np.isnan(u.view(f32))
    assert np.isnan(got.view(f32)[nan]).all()
    bad = np.flatnonzero((got != want) & ~nan)
    assert not len(bad), [(hex(u[i]), hex(got[i]), hex(want[i])) for i in bad[:5]]
    assert got[0] == 0x3f800000 and got[1] == 0x3f820000  # ties to even, down and up
    assert got[15] == 0x7f800000 and got[16] == 0xff800000  # the largest finite float rounds to infinity


def test_reverb_plan_design_figures():
    # DESIGN.md §3 on 132 SMs: config 4 is one wave of 128 tiles of 256 frames; config 5 is 4096 tiles, 31 full waves and a
    # tail of 4 tiles split 33 ways
    assert reverb_plan(256, 2, 8192, 48000, 132) == (256, 128, 0, 1)
    assert reverb_plan(65536, 2, 1024, 48000, 132) == (256, 4096, 4, 33)
    # the shapes of test_gpu_parity.py::test_conv_reverb_many_tiles_vs_fft: 186, 188 and 190 tiles 192 frames wide with a 2-way
    # split, then 1850 tiles 256 frames wide with a 4-way split. (Its docstring's 276 for the first shape is the count at BN = 128,
    # a width that shape never runs.)
    assert reverb_plan(300, 2, 23 * 256, 4100, 132) == (192, 186, 54, 2)
    assert reverb_plan(129, 2, 35 * 256, 4100, 132) == (192, 188, 56, 2)
    assert reverb_plan(520, 2, 14 * 256, 4100, 132) == (192, 190, 58, 2)
    assert reverb_plan(513, 2, 185 * 256, 3850, 132) == (256, 1850, 2, 4)
    # a single wave always picks 128
    assert reverb_plan(130, 2, 777, 4100, 132)[0] == 128


def test_shape_matrix_covers_every_width_and_split():
    m = shape_matrix(132)
    assert sorted(m) == KEYS
    for (bn, sp), (V, C, T, L) in m.items():
        assert reverb_plan(V, C, T, L, 132)[0] == bn and (reverb_plan(V, C, T, L, 132)[3] > 1) == sp
    assert m[(128, True)] == (8449, 2, 128, 2048)


# ---- GPU: every tile width and K-split -------------------------------------------------------------------------------
@pytest.mark.gpu
def test_shape_matrix_on_device(sms):
    m = shape_matrix(sms)
    assert sorted(m) == KEYS, f"{sms} SMs: (BN, split) combinations found: {sorted(m)}"
    print(f"{sms} SMs:", {k: (v, reverb_plan(*v, sms)) for k, v in sorted(m.items())})


@pytest.mark.gpu
@pytest.mark.parametrize("bn,split", KEYS, ids=[f"bn{b}-{'split' if s else 'whole'}" for b, s in KEYS])
def test_impulses_exact_at_every_tile_shape(gpu, sms, bn, split):
    V, C, T, L = shape_matrix(sms)[(bn, split)]
    assert reverb_plan(V, C, T, L, sms)[0] == bn
    lens = [T, T]
    h = reverb_ir(L, 2, L + C)
    x, rows = impulses(V, C, lens, L, call_marks(lens, bn), seed=bn)
    y, _ = stream(gpu, C, h, x, lens, max_call_frames=T)
    assert_equal_samples(y, impulse_answer(rows, V, C, sum(lens), h, L), f"V {V} C {C} T {T} L {L} BN {bn} split {split}")


@pytest.mark.gpu
@pytest.mark.parametrize("bn,split", KEYS, ids=[f"bn{b}-{'split' if s else 'whole'}" for b, s in KEYS])
def test_dense_per_row_at_every_tile_shape(gpu, sms, bn, split):
    V, C, T, L = shape_matrix(sms)[(bn, split)]
    lens = [T, T]
    h = reverb_ir(L, 2, L + 7)
    x, zero = dense(V, C, sum(lens), bn + C)
    y, _ = stream(gpu, C, h, x, lens, max_call_frames=T)
    check_dense(y, x, h, lens, sample_rows(V, C), f"V {V} C {C} T {T} L {L} BN {bn} split {split}", zero)


# ---- GPU: channel map, IR length, history edges ----------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("C", [1, 2, 3])
@pytest.mark.parametrize("ir_ch", [1, 2, 3])
def test_ir_channel_map(gpu, C, ir_ch):
    """Channel c of the node convolves with IR row c % ir_ch; 3 channels go through the generic lowering."""
    V, L, lens = 130, 300, [512, 777, 256]
    h = reverb_ir(L, ir_ch, 10 * C + ir_ch)
    x, rows = impulses(V, C, lens, L, call_marks(lens, 128), seed=C * 3 + ir_ch)
    y, _ = stream(gpu, C, h, x, lens)
    assert_equal_samples(y, impulse_answer(rows, V, C, sum(lens), h, L), f"C {C} ir_ch {ir_ch}")


@pytest.mark.gpu
@pytest.mark.parametrize("L", [1, 2, 8, 9, 64, 65, 4097])
def test_ir_lengths(gpu, L):
    """L - 1 on and off the multiples of 8 (history window start) and 64 (history length); L = 1 has no history at all."""
    V, C, lens = 130, 2, [1000, 8, 1003, 2048]
    h = reverb_ir(L, 2, L)
    x, rows = impulses(V, C, lens, L, call_marks(lens, 128), seed=L)
    y, _ = stream(gpu, C, h, x, lens)
    assert_equal_samples(y, impulse_answer(rows, V, C, sum(lens), h, L), f"impulses, L {L}")
    xd, zero = dense(V, C, sum(lens), L)
    y, _ = stream(gpu, C, h, xd, lens)
    if L == 1:  # one product per sample: exact for dense input too
        want = (bf16_rne(h[:, 0]).astype(np.float64)[None, :, None] * bf16_rne(xd).astype(np.float64)).astype(f32)
        assert_equal_samples(y, want, "dense, L 1")
    else:
        check_dense(y, xd, h, lens, sample_rows(V, C), f"dense, L {L}", zero)


@pytest.mark.gpu
def test_call_lengths_across_both_compactions(gpu, sms):
    """Odd-length calls move the history cursor off the 8-sample grid and the next call compacts the history; the 65536-frame
    call fills the buffer and the call after it compacts because the buffer is full."""
    V, C, L = 130, 2, 4100
    bn = reverb_plan(V, C, 1024, L, sms)[0]
    lens = [1, 7, 8, 777, bn - 1, bn + 1, 65536, 3]
    h = reverb_ir(L, 2, 3)
    x, rows = impulses(V, C, lens, L, call_marks(lens, bn) + list(np.cumsum(lens) - 2), seed=5)
    y, _ = stream(gpu, C, h, x, lens, max_call_frames=65536)
    assert_equal_samples(y, impulse_answer(rows, V, C, sum(lens), h, L), f"impulses, calls {lens}")
    xd, zero = dense(V, C, sum(lens), 6)
    y, _ = stream(gpu, C, h, xd, lens, max_call_frames=65536)
    check_dense(y, xd, h, lens, sample_rows(V, C, n=6), f"dense, calls {lens}", zero)


@pytest.mark.gpu
def test_two_reverbs_in_one_dag_at_a_split_shape(gpu, sms):
    """Two reverb nodes with different L and IR channel counts side by side: each has its own fix-up workspace and epochs."""
    LA, LB = 4100, 2500
    shape = None
    for V in (257, 513, 771, 1030):
        for T in range(4096, 16385, 8):
            pa, pb = reverb_plan(V, 1, T, LA, sms), reverb_plan(V, 1, T, LB, sms)
            if pa[3] > 1 and pb[3] > 1:
                shape = (V, T)
                break
        if shape:
            break
    assert shape, f"no shape splits both reverbs on {sms} SMs"
    V, T = shape
    hA, hB = reverb_ir(LA, 2, 1), reverb_ir(LB, 1, 2)
    lens = [T, T]
    bn = reverb_plan(V, 1, T, LA, sms)[0]
    x, rows = impulses(V, 2, lens, max(LA, LB), call_marks(lens, bn), seed=9)
    cx = FirewheelGraphCtx(gpu, AudioGraphConfig(num_graph_inputs=2, num_graph_outputs=4, num_voices=V, max_call_frames=T))
    g = cx.graph
    ra, rb = g.add_node(2, 2, ConvReverbNode(hA)), g.add_node(2, 2, ConvReverbNode(hB))
    for c in range(2):
        g.connect(g.graph_in_node(), c, ra, c, False); g.connect(g.graph_in_node(), c, rb, c, False)
        g.connect(ra, c, g.graph_out_node(), c, False); g.connect(rb, c, g.graph_out_node(), 2 + c, False)
    proc = cx.activate(SR, 2, 4, 256)
    assert cx.update().graph_error is None, cx.last_error()
    ys = [run_planar(proc, np.ascontiguousarray(x[:, :, k * T:(k + 1) * T]), 4)[0] for k in range(2)]
    close(cx, proc)
    y = np.concatenate(ys, axis=2)
    N = 2 * T
    assert_equal_samples(y[:, :2], impulse_answer(rows, V, 2, N, hA, LA), f"reverb A (L {LA}, 2 IR channels), V {V} T {T}")
    assert_equal_samples(y[:, 2:], impulse_answer(rows, V, 2, N, hB, LB), f"reverb B (L {LB}, 1 IR channel), V {V} T {T}")


@pytest.mark.gpu
@pytest.mark.parametrize("C", [2, 3])
def test_silence_masks_match_oracle(gpu, oracle, C):
    V, L, lens = 5, 200, [512, 300, 512, 256]
    h = reverb_ir(L, 2, 4)
    x, _ = dense(V, C, sum(lens), 8, zero_every=1000)
    x[:, 1] = 0                   # one channel silent throughout
    x[:, :, 512:] = 0              # then the rest rings out and goes silent
    outs = [stream(lib, C, h, x, lens) for lib in (gpu, oracle)]
    assert outs[0][1] == outs[1][1], f"silence masks {[hex(m) for m in outs[0][1]]} != oracle {[hex(m) for m in outs[1][1]]}"
    yo = outs[1][0].reshape(V * C, -1).astype(np.float64)
    assert_close_per_row(outs[0][0].reshape(V * C, -1), yo, lens, f"C {C} vs oracle")


# ---- regressions -----------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("F", [100, 12])
def test_zero_first_block_after_swap_with_reverb_at_stage_0(gpu, oracle, F):
    """After a schedule swap the first block of the caller's rows reads as zero (Q11), also when that block is not a multiple
    of 8 frames and the history is written 8 samples at a time."""
    V, C, L, T = 3, 2, 300, 8 * F
    h = reverb_ir(L, 2, F)
    x, _ = dense(V, C, 3 * T, F, zero_every=1000)
    outs = []
    for lib in (gpu, oracle):
        cx, proc, rv = reverb_ctx(lib, C, h, V, F)
        g = cx.graph
        ys = [run_planar(proc, np.ascontiguousarray(x[:, :, :T]), C)[0]]
        vol = g.add_node(C, C, VolumeNode(100.0))
        for c in range(C):
            assert g.disconnect(rv, c, g.graph_out_node(), c)
            g.connect(rv, c, vol, c, False)
            g.connect(vol, c, g.graph_out_node(), c, False)
        assert cx.update().graph_error is None, cx.last_error()
        ys += [run_planar(proc, np.ascontiguousarray(x[:, :, k * T:(k + 1) * T]), C)[0] for k in (1, 2)]
        close(cx, proc)
        outs.append(np.concatenate(ys, axis=2).reshape(V * C, -1))
    assert_close_per_row(outs[0], outs[1].astype(np.float64), [T, T, T], f"block {F}")
    xz = x.copy()
    xz[:, :, T:T + F] = 0
    ref = ref_conv(xz.reshape(V * C, -1), h[[r % C for r in range(V * C)]])
    assert_close_per_row(outs[0], ref, [T, T, T], f"block {F} vs the input with its first block after the swap zeroed")


@pytest.mark.gpu
@pytest.mark.parametrize("C", [2, 3])
def test_call_longer_than_the_history_buffer(gpu, C):
    """A chunk of more than 65536 frames is processed as consecutive pieces: it gives the same bits as the same input sent as
    two calls cut at the piece boundary."""
    V, L, F, N = 3, 4100, 512, 71680
    h = reverb_ir(L, 2, 11)
    x, zero = dense(V, C, N, 12, zero_every=5)
    y1, _ = stream(gpu, C, h, x, [N], F, 1 << 17)
    y2, _ = stream(gpu, C, h, x, [65536, N - 65536], F, 1 << 17)
    assert_bit_exact(y1, y2, "one call vs two calls")
    check_dense(y1, x, h, [65536, N - 65536], list(range(V * C)), f"C {C}, one call of {N} frames", zero)
