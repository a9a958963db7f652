"""Master bus over more than two graph_out channels (5.1, 7.1; up to FW_MAX_BUS_CHANNELS = 8): the bus is one balanced SumNode tree per
channel, and the device runs it as ceil(C / 2) channel-pair reductions of the chain kernel's bus variant in one launch (grid.z = pair).

CPU (no mark): on the oracle the batched bus equals the flat reference graph with a 2C -> C SumNode tree, and the product's voice
detection turns such a graph into a C-channel bus context. GPU: bit-exact against the oracle, silence masks included, on every path
the bus takes — voices written straight to the caller's bus (<= 64) or through one or two combine levels, the scalar instantiation,
chunked calls (a column window of the caller's bus), sampler sources with fewer channels than the bus, all voices muted, a schedule
swap, the interleaved entry point and the pull stream, a flat graph brought in through detect_voices / new_batched, and two ranks.
Run as a script under torchrun, this file is the worker of the two-rank case."""
import os
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import pytest

from conftest import synth
from firewheel_b200 import AudioGraphConfig, FirewheelGraphCtx, HardClipNode, SamplerNode, SumNode, VolumeNode
from helpers import SR, assert_bit_exact, f32, run_planar

ROOT = Path(__file__).resolve().parent.parent
F = 128


def pairs(C):
    """(first channel, width) of each Volume of a voice: a stereo Volume per channel pair, a mono Volume on an odd last channel"""
    return [(z, min(2, C - z)) for z in range(0, C, 2)]


def voice_gains(C, V, seed):
    rng = np.random.default_rng(seed)
    return [(10 + 140 * rng.random(V)).astype(f32) for _ in pairs(C)]


def activate(cx, n_in, n_out, F_):
    proc = cx.activate(SR, n_in, n_out, F_)
    assert proc is not None
    st = cx.update()
    assert st.kind == "Active" and st.graph_error is None, (st, cx.last_error())
    return proc


def surround(C, V, gains, F_=F, mcf=0):
    """graph_in(C) -> a Volume per channel pair -> graph_out(C) -> master bus; per-voice gains set before activation (no ramp)"""
    def build(lib):
        cx = FirewheelGraphCtx(lib, AudioGraphConfig(num_graph_inputs=C, num_graph_outputs=C, num_voices=V, master_bus=True, max_call_frames=mcf))
        g = cx.graph
        vols = []
        for (z, w), pct in zip(pairs(C), gains):
            vol = g.add_node(w, w, VolumeNode(100.0))
            for c in range(w):
                g.connect(g.graph_in_node(), z + c, vol, c, False)
                g.connect(vol, c, g.graph_out_node(), z + c, False)
            g.set_percent_volume(vol, pct)
            vols.append(vol)
        return cx, activate(cx, C, C, F_), vols
    return build


def stamped(stores):
    """parameter stores at block offsets into the next call: [(block, volume index, percent, voice or None)]; each starts a ramp"""
    def act(cx, vols):
        g = cx.graph
        for block, i, pct, voice in stores:
            g.set_event_block(block)
            if voice is None:
                g.set_percent_volume(vols[i], pct)
            else:
                g.set_percent_volume(vols[i], pct, voice=voice)
        g.set_event_block(0)
    return act


def run_calls(lib, build, calls, C):
    """build(lib) -> (cx, proc, handles); calls: [(x, act or None)], act(cx, handles) runs before its call"""
    cx, proc, h = build(lib)
    res = []
    for x, act in calls:
        if act is not None:
            act(cx, h)
        res.append(run_planar(proc, x, C, True))
    proc.free(); cx.update(); cx.free()
    return res


def compare(gpu, oracle, build, calls, C):
    a, b = run_calls(gpu, build, calls, C), run_calls(oracle, build, calls, C)
    for i, ((yg, mg), (yo, mo)) in enumerate(zip(a, b)):
        assert_bit_exact(yg, yo, f"call {i}")
        assert mg == mo, f"call {i}: silence mask {mg:#x} != {mo:#x}"
    return a


# ---- the flat reference graph: V voices under a 2C -> C SumNode tree (C -> C carries) --------------------------------------------------
def play(g, smp, voice, res):
    g.sampler_set_sample(smp, res, True, voice=voice)
    g.sampler_set_loop_range(smp, "full", voice=voice)
    g.sampler_play(smp, voice=voice)


def flat_graph(lib, C, V, gains, sampled=False):
    """voice v = the per-pair Volumes of surround() with voice v's gains, reading graph_in channels v*C .. v*C + C - 1, or (sampled) a
    SamplerNode(C) of its own: graph_in carries at most 64 channels (FW_MAX_PORTS), so wider flat graphs start each voice at a sampler"""
    cx = FirewheelGraphCtx(lib, AudioGraphConfig(num_graph_inputs=0 if sampled else C * V, num_graph_outputs=C))
    g = cx.graph
    cx.samplers = []  # voice order; flat_calls starts them once the context is active
    level = []
    for v in range(V):
        ends = []
        if sampled:
            smp = g.add_node(0, C, SamplerNode(100.0))
            cx.samplers.append(smp)
        for (z, w), pct in zip(pairs(C), gains):
            vol = g.add_node(w, w, VolumeNode(float(pct[v])))
            for c in range(w):
                g.connect(*((smp, z + c) if sampled else (g.graph_in_node(), v * C + z + c)), vol, c, False)
            ends += [(vol, c) for c in range(w)]
        level.append(ends)
    while len(level) > 1:
        nxt = []
        for i in range(0, len(level) - 1, 2):
            s = g.add_node(2 * C, C, SumNode())
            for c in range(C):
                g.connect(*level[i][c], s, c, False)
                g.connect(*level[i + 1][c], s, C + c, False)
            nxt.append([(s, c) for c in range(C)])
        if len(level) % 2:
            s = g.add_node(C, C, SumNode())
            for c in range(C):
                g.connect(*level[-1][c], s, c, False)
            nxt.append([(s, c) for c in range(C)])
        level = nxt
    for c in range(C):
        g.connect(*level[0][c], g.graph_out_node(), c, False)
    return cx


def sample_resources(g, C):
    return [g.create_sample_resource(synth((ch, 2000 + 97 * i), 80 + i)) for i, ch in enumerate((C, 1, 2))]


def flat_calls(lib, C, V, gains, xs, sampled=False):
    cx = flat_graph(lib, C, V, gains, sampled)
    n_in = 0 if sampled else C * V
    proc = activate(cx, n_in, C, F)
    res = sample_resources(cx.graph, C)
    for v, smp in enumerate(cx.samplers):
        play(cx.graph, smp, 0, res[v % len(res)])
    res = [run_planar(proc, x.reshape(1, n_in, x.shape[-1]), C, False) for x in xs]
    proc.free(); cx.update(); cx.free()
    return [(y[0], m) for y, m in res]


def sampled_surround(C, V, gains):
    """the batched form of flat_graph(sampled=True): graph_in(0) -> SamplerNode(C) -> a Volume per channel pair -> graph_out(C) -> bus"""
    def build(lib):
        cx = FirewheelGraphCtx(lib, AudioGraphConfig(num_graph_inputs=0, num_graph_outputs=C, num_voices=V, master_bus=True))
        g = cx.graph
        smp = g.add_node(0, C, SamplerNode(100.0))
        for (z, w), pct in zip(pairs(C), gains):
            vol = g.add_node(w, w, VolumeNode(100.0))
            for c in range(w):
                g.connect(smp, z + c, vol, c, False)
                g.connect(vol, c, g.graph_out_node(), z + c, False)
            g.set_percent_volume(vol, pct)
        proc = activate(cx, 0, C, F)
        res = sample_resources(g, C)
        for v in range(V):
            play(g, smp, v, res[v % len(res)])
        return cx, proc, None
    return build


def surround_inputs(C, V, seed):
    xs = [synth((V, C, 5 * F + 9), seed), synth((V, C, 3 * F), seed + 1)]
    xs[0][V // 2] = 0.0  # a silent voice: the tree sees flagged inputs
    xs[0][:, C - 1, F: 2 * F] = -0.0
    return xs


@pytest.mark.parametrize("C", [3, 6, 8])
@pytest.mark.parametrize("V", [2, 5, 13])
def test_bus_equals_the_flat_graph_on_the_oracle(oracle, C, V):
    gains = voice_gains(C, V, 10 * C + V)
    sampled = C * V > 64
    xs = [np.zeros((V, 0, 4 * F + 9), f32)] * 2 if sampled else surround_inputs(C, V, C * V)
    want = flat_calls(oracle, C, V, gains, xs, sampled)
    got = run_calls(oracle, (sampled_surround if sampled else surround)(C, V, gains), [(x, None) for x in xs], C)
    for i, ((yb, mb), (yf, mf)) in enumerate(zip(got, want)):
        assert_bit_exact(yb, yf, f"C={C} V={V} call {i}")


@pytest.mark.parametrize("C", [3, 6, 8])
@pytest.mark.parametrize("V", [2, 5, 13])
def test_detection_builds_a_c_channel_bus_context(product, C, V):
    sampled = C * V > 64
    cx = flat_graph(product, C, V, voice_gains(C, V, 1), sampled)
    t = cx.graph.detect_voices()
    assert (t.num_voices, t.num_template_nodes, t.voice_inputs, t.voice_outputs) == (V, len(pairs(C)) + sampled, 0 if sampled else C, C)
    bcx, tids = FirewheelGraphCtx.new_batched(cx)
    assert bcx.config.master_bus and bcx.config.num_voices == V and bcx.config.num_graph_outputs == C
    bcx.free(); cx.free()


# ---- GPU -------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("C", [3, 4, 5, 6, 8])
@pytest.mark.parametrize("V", [1, 2, 63, 64, 65, 130, 1100])
def test_surround_bus_matches_the_oracle(gpu, oracle, C, V):
    """<= 64 voices: the chain kernel writes the caller's bus; 65 .. 1024: one combine level; 1100: two. Ramps start mid-call."""
    gains = voice_gains(C, V, C + 7 * V)
    T = 5 * F
    x = synth((V, C, T), C * 1000 + V)
    x[V // 2, :, T // 3:] = 0.0
    ramps = stamped([(1, 0, 20.0, None), (3, len(pairs(C)) - 1, 150.0, V - 1), (4, len(pairs(C)) // 2, 0.0, 0)])
    calls = [(x, None), (x, ramps), (x[:, :, :2 * F + 7].copy(), None), (x, stamped([(2, 0, 90.0, None)])), (x, None)]
    compare(gpu, oracle, surround(C, V, gains), calls, C)


@pytest.mark.gpu
@pytest.mark.parametrize("C", [5, 6])
@pytest.mark.parametrize("F_,V,mcf", [(100, 37, 0), (255, 130, 0), (64, 37, 3), (64, 130, 3), (100, 1100, 3)])
def test_scalar_path_and_column_window(gpu, oracle, C, F_, V, mcf):
    """F = 100 / 255 with T = 777: the VEC = 1 instantiation. max_call_frames of 3 blocks: every call is chunked, and the bus is a
    column window of the caller's rows, written by the chain kernel (<= 64 voices) or the last combine level"""
    gains = voice_gains(C, V, 3 * V)
    x = synth((V, C, 777), 50 + C)
    calls = [(x, None), (x, stamped([(2, 0, 30.0, None), (5, len(pairs(C)) - 1, 130.0, 1)])), (x, None)]
    compare(gpu, oracle, surround(C, V, gains, F_=F_, mcf=mcf * F_), calls, C)


def sampler_bus(V, res_channels, F_=F):
    """graph_in(0) -> SamplerNode(6) -> Volume(6) -> graph_out(6) -> bus; voice v plays a resource of res_channels[v % n] channels: the
    sampler zeroes and flags the channels the resource lacks, and Volume(6)'s body depends on those flags"""
    def build(lib):
        cx = FirewheelGraphCtx(lib, AudioGraphConfig(num_graph_inputs=0, num_graph_outputs=6, num_voices=V, master_bus=True))
        g = cx.graph
        smp, vol = g.add_node(0, 6, SamplerNode(90.0)), g.add_node(6, 6, VolumeNode(100.0))
        for c in range(6):
            g.connect(smp, c, vol, c, False); g.connect(vol, c, g.graph_out_node(), c, False)
        g.set_percent_volume(vol, (40 + np.arange(V) % 7 * 15).astype(f32))
        proc = activate(cx, 0, 6, F_)
        res = [g.create_sample_resource(synth((ch, 3000 + 111 * i), 70 + i)) for i, ch in enumerate(res_channels)]
        for v in range(V):
            g.sampler_set_sample(smp, res[v % len(res)], True, voice=v)
            g.sampler_set_loop_range(smp, "full", voice=v)
        g.sampler_play(smp)
        return cx, proc, [vol]
    return build


@pytest.mark.gpu
@pytest.mark.parametrize("V", [3, 70])
def test_sampler_source_with_fewer_channels_than_the_bus(gpu, oracle, V):
    z = np.zeros((V, 0, 4 * F), f32)
    calls = [(z, None), (z, stamped([(1, 0, 10.0, None), (2, 0, 120.0, 0)])), (np.zeros((V, 0, 2 * F + 5), f32), None), (z, None)]
    compare(gpu, oracle, sampler_bus(V, [1, 2, 6]), calls, 6)


@pytest.mark.gpu
@pytest.mark.parametrize("V", [5, 130])
def test_mono_source_through_a_gain_matrix(gpu, oracle, V):
    """graph_in(1) -> eight mono Volumes (one gain per output channel) -> graph_out(8) -> bus"""
    rng = np.random.default_rng(V)
    gains = [(150 * rng.random(V)).astype(f32) for _ in range(8)]

    def build(lib):
        cx = FirewheelGraphCtx(lib, AudioGraphConfig(num_graph_inputs=1, num_graph_outputs=8, num_voices=V, master_bus=True))
        g = cx.graph
        vols = []
        for c in range(8):
            vol = g.add_node(1, 1, VolumeNode(100.0))
            g.connect(g.graph_in_node(), 0, vol, 0, False); g.connect(vol, 0, g.graph_out_node(), c, False)
            g.set_percent_volume(vol, gains[c])
            vols.append(vol)
        return cx, activate(cx, 1, 8, F), vols
    x = synth((V, 1, 4 * F + 3), 90)
    compare(gpu, oracle, build, [(x, None), (x, stamped([(1, 3, 0.0, None), (2, 7, 60.0, V - 1)])), (x, None)], 8)


@pytest.mark.gpu
@pytest.mark.parametrize("C", [3, 6, 8])
def test_all_voices_muted(gpu, oracle, C):
    V = 130
    gains = [np.zeros(V, f32) for _ in pairs(C)]
    x = synth((V, C, 3 * F), 5)
    for y, m in compare(gpu, oracle, surround(C, V, gains), [(x, None), (x, None)], C):
        assert m == (1 << C) - 1
        assert not np.any(y.view(np.uint32)), "every sample of a silent bus is +0.0"


@pytest.mark.gpu
def test_schedule_swap_between_six_channel_bus_graphs(gpu, oracle):
    """a HardClipNode(6) spliced in before graph_out and taken out again: the first block after each swap reads zero inputs (Q11)"""
    C, V = 6, 70
    gains = voice_gains(C, V, 2)
    base = surround(C, V, gains)

    def build(lib):
        cx, proc, vols = base(lib)
        return cx, proc, {"vols": vols}

    def splice(cx, h):
        g = cx.graph
        clip = g.add_node(C, C, HardClipNode(-4.0))
        for (z, w), vol in zip(pairs(C), h["vols"]):
            for c in range(w):
                assert g.disconnect(vol, c, g.graph_out_node(), z + c)
                g.connect(vol, c, clip, z + c, False)
        for c in range(C):
            g.connect(clip, c, g.graph_out_node(), c, False)
        assert cx.update().graph_error is None, cx.last_error()
        h["clip"] = clip

    def unsplice(cx, h):
        g = cx.graph
        g.remove_node(h.pop("clip"))
        for (z, w), vol in zip(pairs(C), h["vols"]):
            for c in range(w):
                g.connect(vol, c, g.graph_out_node(), z + c, False)
        assert cx.update().graph_error is None, cx.last_error()
    x = synth((V, C, 3 * F), 8)
    compare(gpu, oracle, build, [(x, None), (x, splice), (x, None), (x, unsplice), (x, None)], C)


@pytest.mark.gpu
def test_interleaved_entry_point(gpu, oracle):
    C, V, T = 6, 70, 3 * F + 40
    gains = voice_gains(C, V, 4)
    x = synth((V, T, C), 12)  # [voice][frame][channel]
    outs = []
    for lib in (gpu, oracle):
        cx, proc, _ = surround(C, V, gains)(lib)
        res = []
        for _ in range(2):
            y = np.full((T, C), np.nan, f32)
            assert proc.process_interleaved(x, y, C, C, T) == 0
            res.append(y)
        proc.free(); cx.update(); cx.free()
        outs.append(res)
    for i, (yg, yo) in enumerate(zip(*outs)):
        assert_bit_exact(yg, yo, f"call {i}")


@pytest.mark.gpu
def test_pull_stream_on_a_six_channel_bus(gpu, oracle):
    """what the consumer pulls equals the oracle's process_interleaved, period by period"""
    V, period, n_periods = 9, 384, 6
    build = sampler_bus(V, [2, 6, 1])
    cx, proc, _ = build(gpu)
    st = proc.open_stream(6, SR, period, ring_periods=4)
    assert st is not None, gpu.last_device_error()
    got, pulled, total = [], 0, period * n_periods
    for n in [100, 383, 384, 700, 5, 64] * 10:
        n = min(n, total - pulled)
        if n == 0:
            break
        t0 = time.time()
        while st.frames_ready() < n:
            assert time.time() - t0 < 10.0, "producer thread made no progress"
            time.sleep(0.001)
        y, k, status, _ = st.pull(n)
        assert k == n and status == 0
        got.append(y); pulled += n
    st.close()
    proc.free(); cx.update(); cx.free()
    cx, proc, _ = build(oracle)
    want = []
    for _ in range(n_periods):
        out = np.full((period, 6), np.nan, f32)
        assert proc.process_interleaved(np.zeros(0, f32), out, 0, 6, period) == 0
        want.append(out)
    proc.free(); cx.update(); cx.free()
    assert_bit_exact(np.concatenate(got), np.concatenate(want), "pulled")


@pytest.mark.gpu
@pytest.mark.parametrize("V", [5, 70])
def test_flat_graph_through_detection_runs_on_the_device(gpu, oracle, V):
    """70 voices do not fit graph_in's 64 channels: each voice then starts at its own SamplerNode(6)"""
    C = 6
    sampled = C * V > 64
    gains = voice_gains(C, V, 21)
    xs = [np.zeros((V, 0, 4 * F + 9), f32)] * 2 if sampled else surround_inputs(C, V, 600 + V)
    want = flat_calls(oracle, C, V, gains, xs, sampled)
    flat = flat_graph(gpu, C, V, gains, sampled)
    bcx, tids = FirewheelGraphCtx.new_batched(flat)
    proc = activate(bcx, 0 if sampled else C, C, F)
    if sampled:
        smp = [t for t in tids if bcx.graph.node_info(t).debug_name in ("beep_test", b"beep_test")]
        res = sample_resources(bcx.graph, C)
        for v in range(V):
            play(bcx.graph, smp[0], v, res[v % len(res)])
    for i, x in enumerate(xs):
        y, m = run_planar(proc, x, C, True)
        assert_bit_exact(y, want[i][0], f"V={V} call {i}")
        assert m == want[i][1]
    proc.free(); bcx.update(); bcx.free(); flat.free()


@pytest.mark.gpu
def test_nine_channels_are_refused(gpu):
    C, V = 9, 4
    cx = FirewheelGraphCtx(gpu, AudioGraphConfig(num_graph_inputs=C, num_graph_outputs=C, num_voices=V, master_bus=True))
    g = cx.graph
    for (z, w) in pairs(C):
        vol = g.add_node(w, w, VolumeNode(100.0))
        for c in range(w):
            g.connect(g.graph_in_node(), z + c, vol, c, False); g.connect(vol, c, g.graph_out_node(), z + c, False)
    proc = cx.activate(SR, C, C, F)
    st = cx.update()
    assert st.graph_error is not None and st.graph_error.kind == "UnsupportedOnDevice"
    assert "more than 8" in cx.last_error()
    out = np.full((C, F), np.nan, f32)
    rc, _ = proc.process_planar(synth((V, C, F), 1), out, C, C, F)
    assert rc == 0 and np.all(out == 0)
    proc.free(); cx.update(); cx.free()


@pytest.mark.gpu
def test_launches_per_call_at_1100_voices_and_eight_channels(gpu):
    """control + 4 stereo Volumes reading the caller's rows (graph_in folded) + the bus launch + 2 combine levels; the first call
    launches kernel by kernel, the third replays the CUDA graph captured by the second"""
    C, V = 8, 1100
    cx, proc, _ = surround(C, V, voice_gains(C, V, 0))(gpu)
    x = synth((V, C, 4 * F), 5)
    deltas = []
    for _ in range(3):
        l0 = proc.kernel_launches()
        run_planar(proc, x, C, True)
        deltas.append(proc.kernel_launches() - l0)
    proc.free(); cx.update(); cx.free()
    assert (deltas[0], deltas[2]) == (8, 8)


@pytest.mark.gpu
def test_six_channel_bus_across_two_ranks(gpu):
    if gpu.device_count() < 2:
        pytest.skip("needs at least 2 GPUs")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
                        "--master-port", "29788", str(Path(__file__).resolve())], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    assert "surround multigpu parity OK" in r.stdout


def _rank_main():
    """one rank of test_six_channel_bus_across_two_ranks: this rank's voices on its GPU, the bus exchanged over NCCL, checked against the
    oracle's tree of the per-rank trees"""
    import firewheel_b200 as fw
    import pyoracle
    from firewheel_b200 import rendezvous
    from sharding import tree_sum, voice_range
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    gpu, oracle = fw.load(), pyoracle.load()
    C, V, T = 6, 201, 4 * F
    gains = voice_gains(C, V, 9)
    x = synth((V, C, T), 31)

    def build(lib, a, b, device=0):
        cx = FirewheelGraphCtx(lib, AudioGraphConfig(num_graph_inputs=C, num_graph_outputs=C, num_voices=b - a, master_bus=True, device=device))
        g = cx.graph
        for (z, w), pct in zip(pairs(C), gains):
            vol = g.add_node(w, w, VolumeNode(100.0))
            for c in range(w):
                g.connect(g.graph_in_node(), z + c, vol, c, False); g.connect(vol, c, g.graph_out_node(), z + c, False)
            g.set_percent_volume(vol, pct[a:b])
        return cx, activate(cx, C, C, F)
    lo, hi = voice_range(V, rank, world)
    cx, proc = build(gpu, lo, hi, device=local)
    rendezvous.init_comm(gpu, proc, rank, world)
    out = np.zeros((C, T), f32)
    for _ in range(2):
        rc, _ = proc.process_planar(np.ascontiguousarray(x[lo:hi]), out, C, C, T)
        assert rc == 0, (rc, gpu.last_device_error())
    parts = []
    for r in range(world):
        a, b = voice_range(V, r, world)
        ocx, oproc = build(oracle, a, b)
        y = np.zeros((C, T), f32)
        for _ in range(2):
            oproc.process_planar(np.ascontiguousarray(x[a:b]), y, C, C, T)
        parts.append(y.copy())
        oproc.free(); ocx.update(); ocx.free()
    ok = np.array_equal(out.view(np.uint32), tree_sum(parts).view(np.uint32))
    all_ok = bool(proc.comm_allgather(np.array([1 if ok else 0], np.int64)).min() == 1)
    proc.comm_allgather(np.zeros(1, np.int64))  # barrier: nobody tears its mailbox down while a peer still runs
    proc.free(); cx.update(); cx.free()
    rendezvous.cleanup(rank)
    if rank == 0:
        print("surround multigpu parity", "OK" if all_ok else "MISMATCH", f"world={world} voices={V} channels={C}")
    sys.exit(0 if all_ok else 1)


if __name__ == "__main__":
    _rank_main()
