"""The temporal kernel family (temporal.cu): biquad cascade, SVF cascade and delay line, against the oracle and exact answers.

launch_temporal sends each pass to one of 61 `biquad_delay_lanes<NS, L, DELAY, FULL, SVF, CHF>` instantiations or to one of the two
scalar kernels. `temporal_kernels` below restates that dispatch, and `stream_kernels` restates where the runtime cuts a call into
passes (host pieces of max_call_frames, chunks at block-stamped commands, the ring cursor after each chunk), so that:
- CPU: the union of the kernels the test matrix reaches equals the set of temporal kernels in the built library;
- GPU: every kernel the restatement predicts for a case shows up in torch.profiler's CUDA activities for that case;
- GPU: the output is bit-identical to the oracle (silence masks included) and, with known-answer coefficients, to a closed form.
The tests without a `gpu` mark also pin a numpy restatement of the three recurrences bit for bit against the oracle."""
import os
import re
import shutil
import subprocess
from collections import namedtuple
from pathlib import Path

import numpy as np
import pytest

from conftest import synth
from firewheel_b200 import (AudioGraphConfig, BiquadNode, DelayNode, FirewheelGraphCtx, HardClipNode, SumNode, SvfNode, design_rbj,
                            design_svf)
from helpers import assert_bit_exact, chain, f32, run_planar

SR = 48000
LANES = (1, 1, 2, 4, 4, 8, 8, 8, 8)  # lanes per row for ns = 0 .. 8 (launch_temporal's switch)
GENERIC, SVF_GENERIC = "biquad_delay_generic", "svf_generic"
Launch = namedtuple("Launch", "kernel ctas row_base")


# ---- the dispatch, restated --------------------------------------------------------------------------------------------
def fast_path(T, zero_first, D, pos, aligned, in_pitch, out_pitch):
    """temporal_fast_path: `aligned` is whether in, out, in2, out2 and the ring all lie on 16 bytes."""
    if T == 0 or T % 32 or zero_first % 32 or not aligned or (in_pitch | out_pitch) % 4:
        return False
    return not (D and (D % 32 or pos % 32 or D < 160))


def lanes_launches(ns, svf, delay, T, zero_first, D, R):
    """launch_lanes + launch_lanes_c: full CTAs of 32 / L rows (64-frame chunks where the shape allows), then the ragged CTA."""
    L = LANES[ns]
    chf = 64 if L in (2, 4) and T % 64 == 0 and zero_first % 64 == 0 and (not delay or D >= 320) else 32
    rows = 32 // L
    full = R // rows
    out = []
    if full:
        out.append(Launch((ns, L, delay, True, svf, chf), full, 0))
    if full * rows < R:
        out.append(Launch((ns, L, delay, False, svf, 32), -(-(R - full * rows) // rows), full * rows))
    return out


def temporal_launches(kind, ns, D, T, zero_first=0, pos=0, R=1, aligned=True, in_pitch=0, out_pitch=0):
    """launch_temporal for one pass. kind: 'biquad' (a lone delay is a biquad pass with ns = 0) or 'svf'."""
    if R == 0 or T == 0:
        return []
    ns = min(ns, 8)
    fast = fast_path(T, zero_first, D, pos, aligned, in_pitch or T, out_pitch or T)
    if kind == "svf":
        return lanes_launches(ns, True, False, T, zero_first, 0, R) if ns >= 1 and D == 0 and fast else [Launch(SVF_GENERIC, -(-R // 64), 0)]
    return lanes_launches(ns, False, D > 0, T, zero_first, D, R) if fast else [Launch(GENERIC, -(-R // 64), 0)]


def temporal_kernels(kind, ns, D, T, zero_first=0, pos=0, R=1, aligned=True, in_pitch=0, out_pitch=0):
    """The kernels one pass of R rows launches, in launch order."""
    return [l.kernel for l in temporal_launches(kind, ns, D, T, zero_first, pos, R, aligned, in_pitch, out_pitch)]


def step_kernels(kind, ns, D, V, blocks, T, zero_first=0, pos=0):
    """run_temporal: `blocks` lists the step's row blocks of V voices as (C, aligned, in_pitch, out_pitch); two consecutive blocks
    share a pass as its two row segments (the pass takes the first block's pitches), and every pass starts at the same cursor."""
    out = []
    for i in range(0, len(blocks), 2):
        seg = blocks[i:i + 2]
        C, _, ip, op = seg[0]
        out += temporal_kernels(kind, ns, D, T, zero_first, pos, len(seg) * V * C, all(b[1] for b in seg), ip, op)
    return out


Call = namedtuple("Call", "T stamps swap last", defaults=((), False, True))


def stream_kernels(kind, ns, D, V, C, F, calls, max_call_frames=0):
    """Kernels per call of a fused chain whose temporal stage is its first stage (it reads the caller's rows through the staging
    buffers of process_planar). Call.stamps: blocks of this call at which a block-stamped command takes effect (later blocks carry
    over to the next call); Call.swap: a schedule swap is picked up at the call's start (Q11); Call.last: the temporal stage writes
    the caller's rows (else a scratch buffer, pitch = chunk length). Restates fw_processor_process_planar (host pieces),
    proc_call (chunks) and run_temporal (the ring cursor)."""
    mcf = -(-(max_call_frames or 64 * F) // F) * F
    pos, pending, per_call, zf_pending = 0, [], [], False
    for call in calls:
        pending += list(call.stamps)
        zf_pending = zf_pending or call.swap
        ks, t0 = [], 0
        while t0 < call.T:
            Tp = min(call.T - t0, mcf)
            nb = -(-Tp // F)
            cuts = sorted({b for b in pending if 0 < b < nb})
            for b0, b1 in zip([0] + cuts, cuts + [nb]):
                c0, Tc = b0 * F, min(Tp, b1 * F) - b0 * F
                zf = min(F, Tc) if zf_pending else 0
                zf_pending = False
                # the staging buffers start on 256 bytes and the chunk's window c0 floats in; scratch rows start on 256 bytes
                ks += temporal_kernels(kind, ns, D, Tc, zf, pos, V * C, c0 % 4 == 0, Tp, Tp if call.last else Tc)
                if D:
                    pos = (pos + Tc) % D
            pending = [b - nb for b in pending if b >= nb]
            t0 += Tp
        per_call.append(ks)
    return per_call, pos


# ---- kernel names ------------------------------------------------------------------------------------------------------
_MANGLED = re.compile(r"biquad_delay_lanesILi(\d+)ELi(\d+)ELb([01])ELb([01])ELb([01])ELi(\d+)E")
_DEMANGLED = re.compile(r"biquad_delay_lanes<([^<>]*)>")


def _arg(t):
    t = re.sub(r"^\(\w+\)", "", t.strip())
    return {"true": 1, "false": 0}[t] if t in ("true", "false") else int(t.rstrip("uUlL"))


def parse_kernel(name):
    """A temporal kernel's key from its mangled or demangled name: (NS, L, DELAY, FULL, SVF, CHF) or a scalar kernel's name; None
    for any other kernel."""
    if GENERIC in name:
        return GENERIC
    if SVF_GENERIC in name:
        return SVF_GENERIC
    m = _MANGLED.search(name)
    args = m.groups() if m else (_DEMANGLED.search(name).group(1).split(",") if _DEMANGLED.search(name) else None)
    if args is None:
        return None
    ns, L, delay, full, svf, chf = (_arg(a) for a in args)
    return (ns, L, bool(delay), bool(full), bool(svf), chf)


def _cuda_tool(name):
    for cand in (shutil.which(name), *(Path(d) / "bin" / name for d in (os.environ.get("CUDA_HOME", ""), os.environ.get("CUDA_PATH", ""), "/usr/local/cuda") if d)):
        if cand and Path(cand).is_file():
            return str(cand)
    return None


def library_kernels(lib_path):
    """The temporal kernels compiled into the library: cuobjdump -symbols, demangled by cu++filt when it is there."""
    dump = _cuda_tool("cuobjdump")
    out = subprocess.run([dump, "-symbols", str(lib_path)], capture_output=True, text=True, check=True).stdout
    names = [ln.split()[-1] for ln in out.splitlines() if "STT_FUNC" in ln and ("biquad_delay" in ln or SVF_GENERIC in ln)]
    filt = _cuda_tool("cu++filt")
    if filt:
        names = subprocess.run([filt], input="\n".join(names), capture_output=True, text=True, check=True).stdout.splitlines()
    return {parse_kernel(n) for n in names} - {None}


# ---- the recurrences, restated (include/fw_b200.h, temporal.cu's header): every op one rounded f32 op ---------------------
def ref_biquad(x, co, st):
    """x [R][N], co [R][ns][5] = {b0, b1, b2, a1, a2}, st [R][ns][2] = {s1, s2} (carried: updated in place)."""
    y = np.empty_like(x)
    b0, b1, b2, a1, a2 = (np.ascontiguousarray(co[:, :, k].T) for k in range(5))
    s1, s2 = np.ascontiguousarray(st[:, :, 0].T), np.ascontiguousarray(st[:, :, 1].T)
    for n in range(x.shape[1]):
        v = x[:, n]
        for s in range(co.shape[1]):
            o = b0[s] * v + s1[s]
            s1[s] = (b1[s] * v - a1[s] * o) + s2[s]
            s2[s] = b2[s] * v - a2[s] * o
            v = o
        y[:, n] = v
    st[:, :, 0], st[:, :, 1] = s1.T, s2.T
    return y


def ref_svf(x, co, st):
    """co [R][ns][6] = {a1, a2, a3, m0, m1, m2}, st [R][ns][2] = {ic1, ic2}:
    v3 = x - ic2;  v1 = a1*ic1 + a2*v3;  v2 = ic2 + (a2*ic1 + a3*v3);  ic1 = 2*v1 - ic1;  ic2 = 2*v2 - ic2;  y = m0*x + (m1*v1 + m2*v2)."""
    y = np.empty_like(x)
    a1, a2, a3, m0, m1, m2 = (np.ascontiguousarray(co[:, :, k].T) for k in range(6))
    ic1, ic2 = np.ascontiguousarray(st[:, :, 0].T), np.ascontiguousarray(st[:, :, 1].T)
    two = f32(2.0)
    for n in range(x.shape[1]):
        v = x[:, n]
        for s in range(co.shape[1]):
            v3 = v - ic2[s]
            v1 = a1[s] * ic1[s] + a2[s] * v3
            v2 = ic2[s] + (a2[s] * ic1[s] + a3[s] * v3)
            ic1[s] = two * v1 - ic1[s]
            ic2[s] = two * v2 - ic2[s]
            v = m0[s] * v + (m1[s] * v1 + m2[s] * v2)
        y[:, n] = v
    st[:, :, 0], st[:, :, 1] = ic1.T, ic2.T
    return y


class RefDelay:
    """Integer delay line: ring [R][D] and one cursor; sample n of a call reads slot (pos + n) % D, then writes x[n] there."""

    def __init__(self, R, D):
        self.D, self.pos, self.ring = D, 0, np.zeros((R, max(D, 1)), f32)

    def process(self, x):
        if self.D == 0:
            return x.copy()
        D, T = self.D, x.shape[1]
        full = np.concatenate([self.ring[:, (self.pos + np.arange(D)) % D], x], axis=1)  # the values slot (pos + k) % D holds, in order
        self.ring[:, (self.pos + T + np.arange(D)) % D] = full[:, T:T + D]
        self.pos = (self.pos + T) % D
        return full[:, :T].copy()


class RefTemporal:
    """One temporal stage (kind, ns, D) over the rows of V voices x C channels; coefficient row of data row r is r // C."""

    def __init__(self, kind, co, D, V, C):
        self.kind, self.D = kind, D
        self.co = np.repeat(co, C, axis=0) if co is not None else None
        self.st = np.zeros((V * C, co.shape[1] if co is not None else 0, 2), f32)
        self.dl = RefDelay(V * C, D)

    def process(self, x):
        if self.co is not None and self.co.shape[1]:
            x = (ref_svf if self.kind == "svf" else ref_biquad)(x, self.co, self.st)
        return self.dl.process(x)


# ---- coefficients and inputs -------------------------------------------------------------------------------------------
def rbj_coeffs(lib, V, ns, seed):
    """Distinct per voice and per stage: lowpass / highpass / peaking / shelves across the band."""
    rng = np.random.default_rng(seed)
    co = np.zeros((V, ns, 5), f32)
    for v in range(V):
        for s in range(ns):
            co[v, s] = design_rbj(lib, int(rng.choice([0, 1, 4, 5, 6])), float(80 * 2 ** rng.uniform(0, 7)), float(rng.uniform(0.5, 2.0)),
                                  float(rng.uniform(-9, 9)), SR)
    return co


def svf_coeffs(lib, V, ns, seed):
    rng = np.random.default_rng(seed)
    co = np.zeros((V, ns, 6), f32)
    for v in range(V):
        for s in range(ns):
            co[v, s] = design_svf(lib, int(rng.integers(0, 6)), float(80 * 2 ** rng.uniform(0, 7)), float(rng.uniform(0.5, 2.0)), SR)
    return co


def kat_coeffs(kind, V, ns, seed):
    """Known-answer stages: biquad stage (v, s) is g[v, s] * x[n - d[v, s]] (one nonzero b, a power of two, at tap d in {0, 1, 2};
    a1 = a2 = 0); SVF stage (v, s) is g[v, s] * x (a1 = a2 = a3 = 0, m1 and m2 multiply zeros). Returns the coefficients, the total
    shift S[v] and the total gain G[v] of each voice."""
    rng = np.random.default_rng(seed)
    g = (rng.choice([-1.0, 1.0], (V, ns)) * 2.0 ** rng.integers(-1, 2, (V, ns))).astype(f32)
    if kind == "svf":
        co = np.zeros((V, ns, 6), f32)
        co[..., 3] = g
        co[..., 4:] = rng.uniform(-1, 1, (V, ns, 2))
        d = np.zeros((V, ns), int)
    else:
        co = np.zeros((V, ns, 5), f32)
        d = rng.integers(0, 3, (V, ns))
        np.put_along_axis(co, d[..., None], g[..., None], axis=2)
    return co, d.sum(axis=1), np.prod(g.astype(np.float64), axis=1)


def closed_form(x, S, G, D):
    """y[v, c, n] = G[v] * x[v, c, n - S[v] - D], zero before the stream starts."""
    V, C, N = x.shape
    y = np.zeros_like(x)
    for v in range(V):
        k = int(S[v]) + D
        if k < N:
            y[v, :, k:] = (G[v] * x[v, :, :N - k].astype(np.float64)).astype(f32)
    return y


def assert_same_values(got, want, what):
    """value equality (+0 == -0), no NaN anywhere"""
    assert not np.isnan(got).any(), f"{what}: NaN in the output"
    bad = np.argwhere(got != want)
    if len(bad):
        i = tuple(bad[0])
        raise AssertionError(f"{what}: {len(bad)} of {got.size} samples differ; first at (voice, channel, frame) {i}: got {got[i]!r} want {want[i]!r}")


# ---- running a chain on any implementation of the C ABI -----------------------------------------------------------------
def temporal_nodes(kind, ns, D):
    """(kind biquad, ns 0, D 0) is DelayNode(0); (biquad, 0, D) a lone DelayNode; a delay after a biquad joins its pass."""
    if kind == "svf":
        return [(SvfNode(ns), 2, 2)]
    nodes = [(BiquadNode(ns), 2, 2)] if ns else []
    if D or not ns:
        nodes.append((DelayNode(D), 2, 2))
    return nodes


def set_coeffs(g, node, kind, co):
    if kind == "svf":
        g.set_svf_coeffs(node, co)
    else:
        g.set_biquad_coeffs(node, co)


def run_chain(lib, kind, ns, D, co, x, calls, F=256, between=None):
    """graph_in(2) -> temporal stage -> graph_out(2); x [V][2][N] sent as consecutive calls. between(k, cx, ids) runs before call k."""
    V = x.shape[0]
    nodes = temporal_nodes(kind, ns, D)
    setup = (lambda cx, ids: set_coeffs(cx.graph, ids[0], kind, co)) if (co is not None and ns) else None
    cx, proc, ids = chain(lib, 2, nodes, voices=V, max_block=F, setup=setup)
    ys, masks, t0 = [], [], 0
    for k, T in enumerate(calls):
        if between:
            between(k, cx, ids)
        y, m = run_planar(proc, np.ascontiguousarray(x[:, :, t0:t0 + T]), 2)
        ys.append(y); masks.append(m); t0 += T
    replays = proc.graph_replays()  # always 0 on the oracle
    proc.free(); cx.update(); cx.free()
    return np.concatenate(ys, axis=2), masks, replays


def profiled_kernels(fn):
    """Run fn() under torch.profiler with CUDA activities; returns fn's result and the temporal kernels that ran."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        res = fn()
        torch.cuda.synchronize()
    ran = {parse_kernel(e.name) for e in prof.events()} - {None}
    assert ran, "the profiler saw no temporal kernel at all"
    return res, ran


# ---- the test matrix ---------------------------------------------------------------------------------------------------
V_A, F_A = 19, 256  # 38 rows: full CTAs and a ragged CTA for every lane width
A_CALLS = (512, 480, 512, 777, 512)
A_D = 352           # an odd multiple of 32, >= 320: a 64-frame ring chunk wraps between its halves
A_CASES = [("biquad", ns, D) for ns in range(9) for D in (0, A_D)] + [("svf", ns, 0) for ns in range(1, 9)]
B_CALLS = (4096, 480, 4096, 4096, 4096)
B_DS = (96, 128, 161, 160, 192, 288, 320, 352, 12000, 20000)  # scalar / 32-frame / 64-frame; 20000 > the whole stream
B_CASES = [(ns, D, B_CALLS) for ns in (2, 0) for D in B_DS] + [(ns, 160, (2048, 2048)) for ns in (2, 0)]
C_SPLIT = (480, 512, 33, 31, 1024, 64)
C_CASES = [("biquad", 4, 352), ("svf", 3, 0)]
D_CASES = [(F, ns, D) for F in (64, 96, 256) for ns in (2, 4) for D in (0, 352)]


def q11_calls(F):
    """call A (4F); the clip is spliced in: call B (T = F, every chunk zeroed); the clip is taken out: call C (4F, first block zeroed); D"""
    return [Call(4 * F), Call(F, swap=True, last=False), Call(4 * F, swap=True), Call(4 * F)]


def matrix_predictions():
    """(case id, predicted kernels per call) for every case of the GPU tests that runs a fused chain."""
    out = []
    for kind, ns, D in A_CASES:
        out.append((f"a-{kind}{ns}-D{D}", stream_kernels(kind, ns, D, V_A, 2, F_A, [Call(T) for T in A_CALLS])[0]))
    for ns, D, calls in B_CASES:
        out.append((f"b-biquad{ns}-D{D}", stream_kernels("biquad", ns, D, V_A, 2, F_A, [Call(T) for T in calls])[0]))
    for kind, ns, D in C_CASES:
        for calls in ((sum(C_SPLIT),), C_SPLIT):
            out.append((f"c-{kind}{ns}-{len(calls)}", stream_kernels(kind, ns, D, V_A, 2, F_A, [Call(T) for T in calls])[0]))
    for F, ns, D in D_CASES:
        out.append((f"d-F{F}-{ns}-D{D}", stream_kernels("biquad", ns, D, V_A, 2, F, q11_calls(F))[0]))
    return out


# ---- CPU: the dispatch restatement -------------------------------------------------------------------------------------
def test_dispatch_hand_worked_cases():
    # V = 19 stereo voices: R = 38 rows. 4 lanes per row: 8 rows per CTA, 4 full CTAs and a ragged CTA of 6 rows
    assert temporal_launches("biquad", 3, 0, 512, R=38) == [Launch((3, 4, False, True, False, 64), 4, 0), Launch((3, 4, False, False, False, 32), 1, 32)]
    # 8 lanes: 4 rows per CTA, 9 full CTAs and 2 ragged rows; the 8-lane kernel has 32-frame chunks only
    assert temporal_launches("biquad", 8, 0, 512, R=38) == [Launch((8, 8, False, True, False, 32), 9, 0), Launch((8, 8, False, False, False, 32), 1, 36)]
    # 1 lane: 32 rows per CTA; 32 rows make no ragged CTA
    assert temporal_launches("biquad", 1, 0, 512, R=32) == [Launch((1, 1, False, True, False, 32), 1, 0)]
    assert temporal_launches("svf", 2, 0, 480, R=16) == [Launch((2, 2, False, True, True, 32), 1, 0)]  # 480 % 64 == 32
    # delay thresholds: D >= 160 and D % 32 == 0 for the lanes kernel, D >= 320 for 64-frame chunks
    assert temporal_kernels("biquad", 2, 128, 512, R=16) == [GENERIC]
    assert temporal_kernels("biquad", 2, 161, 512, R=16) == [GENERIC]
    assert temporal_kernels("biquad", 2, 160, 512, R=16) == [(2, 2, True, True, False, 32)]
    assert temporal_kernels("biquad", 2, 288, 512, R=16) == [(2, 2, True, True, False, 32)]
    assert temporal_kernels("biquad", 2, 320, 512, R=16) == [(2, 2, True, True, False, 64)]
    assert temporal_kernels("biquad", 4, 352, 512, pos=288, R=8) == [(4, 4, True, True, False, 64)]
    assert temporal_kernels("biquad", 4, 352, 512, pos=9, R=8) == [GENERIC]
    # Q11: 96 zeroed frames keep a 384-frame pass on 32-frame chunks; 64 do not
    assert temporal_kernels("biquad", 4, 0, 384, zero_first=96, R=8) == [(4, 4, False, True, False, 32)]
    assert temporal_kernels("biquad", 4, 0, 384, zero_first=64, R=8) == [(4, 4, False, True, False, 64)]
    # scalar kernels: SVF without stages, a misaligned pointer or pitch, a length off the 32-frame grid
    assert temporal_kernels("svf", 0, 0, 512, R=8) == [SVF_GENERIC]
    assert temporal_kernels("svf", 3, 0, 512, R=8, aligned=False) == [SVF_GENERIC]
    assert temporal_kernels("biquad", 3, 0, 512, R=8, in_pitch=1530) == [GENERIC]
    assert temporal_kernels("biquad", 3, 0, 777, R=8) == [GENERIC]
    # two segments of V = 19 one-channel rows share a pass (38 rows), a third block is a pass of its own
    seg = (1, True, 512, 512)
    assert step_kernels("biquad", 4, 0, 19, [seg, seg, seg], 512) == [
        (4, 4, False, True, False, 64), (4, 4, False, False, False, 32), (4, 4, False, True, False, 64), (4, 4, False, False, False, 32)]


def test_stream_splitting_hand_worked():
    # the ring cursor at the start of each of A_CALLS at D = 352: 0, 160, 288 (pos % 64 == 32), 96, 169 (after 777 frames: off the
    # 32-frame grid)
    ks, pos = stream_kernels("biquad", 4, 352, 19, 2, 256, [Call(T) for T in A_CALLS])
    assert pos == sum(A_CALLS) % 352 == 329
    assert ks[0] == [(4, 4, True, True, False, 64), (4, 4, True, False, False, 32)]
    assert ks[1] == [(4, 4, True, True, False, 32), (4, 4, True, False, False, 32)]
    assert ks[2] == ks[0] and ks[3] == [GENERIC] and ks[4] == [GENERIC]
    assert stream_kernels("biquad", 4, 0, 19, 2, 256, [Call(T) for T in A_CALLS])[0][4] == [(4, 4, False, True, False, 64), (4, 4, False, False, False, 32)]
    # a store stamped at block 3 of a 512-frame call cuts it at frame 192 (64-frame blocks): two 64-frame passes; at block 2 of
    # a 510-frame call the rows' pitch 510 is off the 16-byte grid, so both chunks are scalar
    ks, _ = stream_kernels("biquad", 2, 0, 19, 2, 64, [Call(512, stamps=(3,)), Call(510, stamps=(2,))])
    assert ks[0] == [(2, 2, False, True, False, 64), (2, 2, False, False, False, 32)] * 2
    assert ks[1] == [GENERIC, GENERIC]
    # a stamp beyond the call carries over: block 9 of a 512-frame call (8 blocks of 64) is block 1 of the next
    ks, _ = stream_kernels("biquad", 2, 0, 16, 1, 64, [Call(512, stamps=(9,)), Call(256)])
    assert ks == [[(2, 2, False, True, False, 64)], [(2, 2, False, True, False, 64)] * 2]
    # host pieces of max_call_frames = 256 (whole 64-frame blocks): 1000 frames are 256, 256, 256 and 232
    ks, _ = stream_kernels("biquad", 2, 0, 16, 1, 64, [Call(1000)], max_call_frames=250)
    assert ks == [[(2, 2, False, True, False, 64)] * 3 + [GENERIC]]
    # Q11 zeroes min(F, chunk) leading frames of the first chunk after a swap
    ks, _ = stream_kernels("biquad", 4, 0, 8, 1, 96, q11_calls(96))
    assert ks == [[(4, 4, False, True, False, 64)], [(4, 4, False, True, False, 32)], [(4, 4, False, True, False, 32)], [(4, 4, False, True, False, 64)]]


def test_kernel_name_parsing():
    key = (5, 8, True, False, False, 32)
    assert parse_kernel("_ZN2fw18biquad_delay_lanesILi5ELi8ELb1ELb0ELb0ELi32EEEvNS_12TemporalArgsE") == key
    assert parse_kernel("void fw::biquad_delay_lanes<(int)5, (int)8, (bool)1, (bool)0, (bool)0, (int)32>(fw::TemporalArgs)") == key
    assert parse_kernel("void fw::biquad_delay_lanes<5, 8, true, false, false, 32>(fw::TemporalArgs)") == key
    assert parse_kernel("fw::biquad_delay_generic(fw::TemporalArgs)") == GENERIC
    assert parse_kernel("_ZN2fw11svf_genericENS_12TemporalArgsE") == SVF_GENERIC
    assert parse_kernel("void fw::chain_kernel<true>(fw::ChainArgs)") is None


def test_matrix_covers_every_temporal_kernel_in_the_library(product):
    """A new instantiation without a test case fails here."""
    import firewheel_b200
    if not _cuda_tool("cuobjdump"):
        pytest.skip("cuobjdump (CUDA toolkit) not found: the library's kernel list cannot be read")
    built = library_kernels(firewheel_b200.LIB_PATH)
    reached = set()
    for _, per_call in matrix_predictions():
        for ks in per_call:
            reached |= set(ks)
    assert len(built) == 63, sorted(built, key=str)
    assert reached == built, f"in the library, reached by no case: {sorted(built - reached, key=str)}; predicted but not built: {sorted(reached - built, key=str)}"


# ---- CPU: the restatement against the oracle ---------------------------------------------------------------------------
R_CALLS = (512, 777, 480)


def restated(kind, ns, D, co, x, calls):
    V, C, N = x.shape
    ref = RefTemporal(kind, co if ns else None, D, V, C)
    xs = x.reshape(V * C, N)
    ys, t0 = [], 0
    for T in calls:
        ys.append(ref.process(np.ascontiguousarray(xs[:, t0:t0 + T]))); t0 += T
    return np.concatenate(ys, axis=1).reshape(V, C, N)


@pytest.mark.parametrize("kind,ns,D", [("biquad", ns, 352) for ns in range(9)] + [("biquad", 2, D) for D in (0,) + B_DS] + [("svf", ns, 0) for ns in range(9)])
def test_restatement_matches_oracle(oracle, kind, ns, D):
    V = 5
    co = (svf_coeffs if kind == "svf" else rbj_coeffs)(oracle, V, ns, 100 + ns)
    x = synth((V, 2, sum(R_CALLS)), 7 + ns)
    y, _, _ = run_chain(oracle, kind, ns, D, co, x, R_CALLS)
    assert_bit_exact(restated(kind, ns, D, co, x, R_CALLS), y, f"{kind} ns {ns} D {D}: restatement vs oracle")


def test_known_answer_closed_form_on_the_restatement():
    V = 4
    for kind, ns, D in (("biquad", 8, 161), ("svf", 5, 0)):
        co, S, G = kat_coeffs(kind, V, ns, 3)
        x = synth((V, 2, 900), 3)
        assert_same_values(restated(kind, ns, D, co, x, (300, 600)), closed_form(x, S, G, D), f"{kind} {ns}")


# ---- GPU: every instantiation ran and is right -------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("kind,ns,D", A_CASES, ids=[f"{k}{n}-D{d}" for k, n, d in A_CASES])
def test_every_instantiation_runs_and_matches(gpu, oracle, kind, ns, D):
    x = synth((V_A, 2, sum(A_CALLS)), 1000 + 10 * ns + (D > 0) + (kind == "svf") * 500)
    co = (svf_coeffs if kind == "svf" else rbj_coeffs)(gpu, V_A, ns, 7 * ns + (D > 0)) if ns else None
    (yg, mg, _), ran = profiled_kernels(lambda: run_chain(gpu, kind, ns, D, co, x, A_CALLS))
    predicted = stream_kernels(kind, ns, D, V_A, 2, F_A, [Call(T) for T in A_CALLS])[0]
    want = set(k for ks in predicted for k in ks)
    assert ran == want, f"ran {sorted(ran, key=str)}, predicted {sorted(want, key=str)}"
    yo, mo, _ = run_chain(oracle, kind, ns, D, co, x, A_CALLS)
    assert_bit_exact(yg, yo, f"{kind} ns {ns} D {D} vs oracle")
    assert mg == mo, (mg, mo)
    if ns:
        co, S, G = kat_coeffs(kind, V_A, ns, ns + 50 * (D > 0))
    else:
        S, G = np.zeros(V_A, int), np.ones(V_A)
    yk, _, _ = run_chain(gpu, kind, ns, D, co, x, A_CALLS)
    assert_same_values(yk, closed_form(x, S, G, D), f"{kind} ns {ns} D {D} known answer")


# ---- GPU: delay edges --------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("ns,D,calls", B_CASES, ids=[f"{'biquad2' if n else 'delay'}-D{d}-{len(c)}calls" for n, d, c in B_CASES])
def test_delay_edges_known_answer(gpu, ns, D, calls):
    x = synth((V_A, 2, sum(calls)), D + ns)
    co, S, G = kat_coeffs("biquad", V_A, ns, D) if ns else (None, np.zeros(V_A, int), np.ones(V_A))
    (y, _, _), ran = profiled_kernels(lambda: run_chain(gpu, "biquad", ns, D, co, x, calls))
    predicted = stream_kernels("biquad", ns, D, V_A, 2, F_A, [Call(T) for T in calls])[0]
    assert ran == set(k for ks in predicted for k in ks), (sorted(ran, key=str), predicted)
    assert_same_values(y, closed_form(x, S, G, D), f"ns {ns} D {D}")


# ---- GPU: one stream, two ways of cutting it -----------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("kind,ns,D", C_CASES)
def test_split_invariance(gpu, oracle, kind, ns, D):
    x = synth((V_A, 2, sum(C_SPLIT)), 31 + ns)
    co = (svf_coeffs if kind == "svf" else rbj_coeffs)(gpu, V_A, ns, 5)
    one, m1, _ = run_chain(gpu, kind, ns, D, co, x, (sum(C_SPLIT),))
    many, m2, _ = run_chain(gpu, kind, ns, D, co, x, C_SPLIT)
    assert_bit_exact(many, one, f"{kind} {ns}: calls {C_SPLIT} vs one call")
    yo, mo, _ = run_chain(oracle, kind, ns, D, co, x, C_SPLIT)
    assert_bit_exact(one, yo, f"{kind} {ns}: one call vs oracle")
    assert m2 == mo


# ---- GPU: Q11 on every chunk width -------------------------------------------------------------------------------------
def q11_stream(lib, ns, D, co, x, F):
    """q11_calls(F) with a HardClipNode(40 dB, never reached) spliced in after the temporal stage before call B, removed before C"""
    calls = [c.T for c in q11_calls(F)]
    clip = {}

    def between(k, cx, ids):
        g, last = cx.graph, ids[-1]
        if k == 1:
            clip["id"] = g.add_node(2, 2, HardClipNode(40.0))
            for c in range(2):
                assert g.disconnect(last, c, g.graph_out_node(), c)
                g.connect(last, c, clip["id"], c, False); g.connect(clip["id"], c, g.graph_out_node(), c, False)
            assert cx.update().graph_error is None, cx.last_error()
        elif k == 2:
            g.remove_node(clip["id"])
            for c in range(2):
                g.connect(last, c, g.graph_out_node(), c, False)
            assert cx.update().graph_error is None, cx.last_error()
    return run_chain(lib, "biquad", ns, D, co, x, calls, F=F, between=between)


@pytest.mark.gpu
@pytest.mark.parametrize("F,ns,D", D_CASES, ids=[f"F{F}-biquad{n}-D{d}" for F, n, d in D_CASES])
def test_zeroed_first_block_after_swap(gpu, oracle, F, ns, D):
    V = V_A  # full CTAs: the ragged CTA always runs 32-frame chunks
    x = synth((V, 2, 13 * F), F + ns + D)
    co = rbj_coeffs(gpu, V, ns, F + ns)
    (yg, mg, _), ran = profiled_kernels(lambda: q11_stream(gpu, ns, D, co, x, F))
    predicted = stream_kernels("biquad", ns, D, V, 2, F, q11_calls(F))[0]
    assert ran == set(k for ks in predicted for k in ks), (sorted(ran, key=str), predicted)
    yo, mo, _ = q11_stream(oracle, ns, D, co, x, F)
    assert_bit_exact(yg, yo, f"F {F} ns {ns} D {D} vs oracle")
    assert mg == mo
    ck, S, G = kat_coeffs("biquad", V, ns, F)
    yk, _, _ = q11_stream(gpu, ns, D, ck, x, F)
    xz = x.copy()
    xz[:, :, 4 * F:5 * F] = 0  # call B: all of it
    xz[:, :, 5 * F:6 * F] = 0  # call C: its first block
    assert_same_values(yk, closed_form(xz, S, G, D), f"F {F} ns {ns} D {D} known answer")


# ---- GPU: the generic lowering's two-segment passes --------------------------------------------------------------------
E_NODES = [("biquad", 2, 4), ("biquad", 3, 3), ("svf", 2, 2), ("svf", 3, 5), ("delay", 2, 352), ("delay", 3, 160)]


def dag_stream(lib, V, x, calls, stamps, co, co2):
    """graph_in(3) feeds a 2- and a 3-channel biquad, SVF and delay, channel c of node j reading port (2 - c + j) % 3 (channel 0 of
    the first node reads port 2); a SumNode mixes all six into graph_out(3). stamps[k]: block of call k at which the 2-channel
    biquad and the 3-channel SVF take the coefficients co2 (None: no store)."""
    F = 64
    cx = FirewheelGraphCtx(lib, AudioGraphConfig(num_graph_inputs=3, num_graph_outputs=3, num_voices=V))
    g = cx.graph
    mix = g.add_node(3 * len(E_NODES), 3, SumNode())
    ids = []
    for j, (kind, C, p) in enumerate(E_NODES):
        nd = g.add_node(C, C, BiquadNode(p) if kind == "biquad" else SvfNode(p) if kind == "svf" else DelayNode(p))
        ids.append(nd)
        for c in range(C):
            g.connect(g.graph_in_node(), (2 - c + j) % 3, nd, c, False)
        for c in range(3):
            g.connect(nd, min(c, C - 1), mix, 3 * j + c, False)
        if kind != "delay":
            set_coeffs(g, nd, kind, co[j])
    for c in range(3):
        g.connect(mix, c, g.graph_out_node(), c, False)
    proc = cx.activate(SR, 3, 3, F)
    assert cx.update().graph_error is None, cx.last_error()
    ys, masks, t0 = [], [], 0
    for k, T in enumerate(calls):
        if stamps[k] is not None:
            g.set_event_block(stamps[k])
            set_coeffs(g, ids[0], "biquad", co2[0]); set_coeffs(g, ids[3], "svf", co2[3])
            g.set_event_block(0)
        y, m = run_planar(proc, np.ascontiguousarray(x[:, :, t0:t0 + T]), 3)
        ys.append(y); masks.append(m); t0 += T
    proc.free(); cx.update(); cx.free()
    return np.concatenate(ys, axis=2), masks


@pytest.mark.gpu
@pytest.mark.parametrize("V", [1, 19, 64])
def test_generic_lowering_segments_and_pitched_rows(gpu, oracle, V):
    """Two channels of a node share a pass as its two row segments (a CTA straddles the boundary at V = 19), the third channel is a
    pass with srow_add = 2; the nodes read the caller's rows. A stamped store cuts a call at t0 > 0: rows of pitch 3 * 512 (the
    lanes kernel) and 3 * 510 (off the 16-byte grid: the scalar kernel)."""
    calls, stamps = (512, 512, 510, 512), (3, None, 2, 5)
    x = synth((V, 3, sum(calls)), V)
    mk = lambda seed: [(svf_coeffs if k == "svf" else rbj_coeffs)(gpu, V, p, seed + j) if k != "delay" else None for j, (k, _, p) in enumerate(E_NODES)]
    co, co2 = mk(10), mk(40)
    yg, mg = dag_stream(gpu, V, x, calls, stamps, co, co2)
    yo, mo = dag_stream(oracle, V, x, calls, stamps, co, co2)
    assert_bit_exact(yg, yo, f"V {V}")
    assert mg == mo


# ---- GPU: special values -----------------------------------------------------------------------------------------------
SPECIAL = np.array([0.0, -0.0, 2.0 ** -149, -2.0 ** -149, 2.0 ** -140, -3 * 2.0 ** -137, 2.0 ** -126, -2.0 ** -126, 2.0 ** 20, -2.0 ** 20,
                    2.0 ** -20, -2.0 ** -20], f32)
F_CASES = [("biquad", ns, 0) for ns in (1, 2, 4, 8)] + [("biquad", 4, 352)] + [("svf", ns, 0) for ns in (1, 2, 4, 8)]


def special_input(V, N, seed):
    """Rows of four regimes: subnormals and the smallest normals; +-2^20; +-0 and +-2^-20; every special value mixed."""
    rng = np.random.default_rng(seed)
    x = np.empty((V * 2, N), f32)
    tiny = (rng.integers(-(1 << 24), 1 << 24, (V * 2, N)) * 2.0 ** -150).astype(f32)
    for r in range(V * 2):
        reg = r % 4
        if reg == 0:
            x[r] = np.where(rng.random(N) < 0.3, rng.choice(SPECIAL[2:8], N), tiny[r])
        elif reg == 1:
            x[r] = rng.choice(SPECIAL[8:10], N)
        elif reg == 2:
            x[r] = rng.choice(np.concatenate([SPECIAL[:2], SPECIAL[10:]]), N)
        else:
            x[r] = rng.choice(SPECIAL, N)
    return x.reshape(V, 2, N)


@pytest.mark.gpu
@pytest.mark.parametrize("kind,ns,D", F_CASES, ids=[f"{k}{n}-D{d}" for k, n, d in F_CASES])
def test_special_values(gpu, oracle, kind, ns, D):
    calls = (512, 480, 96)
    x = special_input(V_A, sum(calls), ns)
    co = (svf_coeffs if kind == "svf" else rbj_coeffs)(gpu, V_A, ns, 90 + ns)
    yg, mg, _ = run_chain(gpu, kind, ns, D, co, x, calls)
    yo, mo, _ = run_chain(oracle, kind, ns, D, co, x, calls)
    assert_bit_exact(yg, yo, f"{kind} ns {ns} D {D}")
    assert mg == mo


# ---- GPU: CUDA-graph replay --------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("kind,ns", [("biquad", 4), ("svf", 3), ("biquad", 8)])
def test_block_sized_calls_on_graph_replay(gpu, oracle, kind, ns):
    calls = (256,) * 12
    x = synth((V_A, 2, sum(calls)), 60 + ns)
    co = (svf_coeffs if kind == "svf" else rbj_coeffs)(gpu, V_A, ns, 60)
    yg, mg, replays = run_chain(gpu, kind, ns, 0, co, x, calls)
    assert replays >= 9, f"only {replays} of 12 block-sized calls were replayed from a CUDA graph"
    yo, mo, _ = run_chain(oracle, kind, ns, 0, co, x, calls)
    assert_bit_exact(yg, yo, f"{kind} {ns}")
    assert mg == mo
