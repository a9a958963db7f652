"""Streams whose channel counts differ from graph_in's and graph_out's port counts (schedule.rs:213-287, util.rs:90-147,
processor.rs:122-133). With G_in / G_out the port counts and n_in / n_out the stream's channels:

* S1 n_in < G_in: graph_in ports >= n_in carry +0.0, and downstream they are live zeros, not silent (graph_in's Dummy, Q4);
* S2 n_in > G_in: stream channels >= G_in are ignored;
* S3 n_out > G_out: output channels >= G_out are +0.0 and never flagged silent; on the master bus with two or more voices the tree's
  SumNodes then never see all their inputs flagged, so the bus mask is 0;
* S4 n_out < G_out: graph_out ports >= n_out are not read, and the mask covers n_out channels.

CPU (no mark): known answers of the oracle, derived from those reference lines, and the oracle against tests/pyref.py on mismatched
process_interleaved. GPU: the product bit for bit against the oracle, masks included, on the fused chain, the generic lowering and a
plugin node, with and without the master bus, through every entry point, chunked and block-sized, across a schedule swap that changes
graph_out's port count, and the launches per chunk of the mismatched shapes. Every output buffer starts as NaN, so a row the product
leaves unwritten fails. Run as a script under torchrun, this file is the worker of the two-rank case."""
import os
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

import plugin_fixture as pf
import pyref
from conftest import synth
from firewheel_b200 import (AudioGraphConfig, BiquadNode, FirewheelGraphCtx, HardClipNode, PanNode, SamplerNode, SumNode, SvfNode, VolumeNode,
                            design_rbj, design_svf)
from helpers import SR, assert_bit_exact, f32

ROOT = Path(__file__).resolve().parent.parent
F = 64


def activate(cx, n_in, n_out, F_=F):
    proc = cx.activate(SR, n_in, n_out, F_)
    assert proc is not None
    st = cx.update()
    assert st.kind == "Active" and st.graph_error is None, (st, cx.last_error())
    return proc


def ctx(lib, G_in, G_out, V, bus, mcf=0):
    return FirewheelGraphCtx(lib, AudioGraphConfig(num_graph_inputs=G_in, num_graph_outputs=G_out, num_voices=V, master_bus=bus, max_call_frames=mcf))


def voice_pcts(V, seed, muted=False):
    return np.zeros(V, f32) if muted else (10 + 140 * np.random.default_rng(seed).random(V)).astype(f32)


# ---- graphs: build(lib, n_in, n_out, V, bus, mcf) -> (cx, proc) -------------------------------------------------------------------
def gain_pan(G_in=2, G_out=2, muted=False):
    """graph_in(2) -> Volume(2) -> Pan -> graph_out(2): the fused chain (G_in / G_out other than 2 leave ports unconnected)"""
    def build(lib, n_in, n_out, V, bus, mcf=0):
        cx = ctx(lib, G_in, G_out, V, bus, mcf)
        g = cx.graph
        vol, pn = g.add_node(2, 2, VolumeNode(100.0)), g.add_node(2, 2, PanNode(0.0))
        for c in range(2):
            if c < G_in:
                g.connect(g.graph_in_node(), c, vol, c, False)
            g.connect(vol, c, pn, c, False)
            if c < G_out:
                g.connect(pn, c, g.graph_out_node(), c, False)
        g.set_percent_volume(vol, voice_pcts(V, 1, muted))
        g.set_pan(pn, np.random.default_rng(2).uniform(-1, 1, V).astype(f32))
        return cx, activate(cx, n_in, n_out)
    return build


def sampler_chain(lib, n_in, n_out, V, bus, mcf=0):
    """graph_in(0) -> SamplerNode(2) -> Volume(2) -> graph_out(2): the fused chain headed by a sampler"""
    cx = ctx(lib, 0, 2, V, bus, mcf)
    g = cx.graph
    smp, vol = g.add_node(0, 2, SamplerNode(100.0)), g.add_node(2, 2, VolumeNode(100.0))
    for c in range(2):
        g.connect(smp, c, vol, c, False)
        g.connect(vol, c, g.graph_out_node(), c, False)
    g.set_percent_volume(vol, voice_pcts(V, 3))
    proc = activate(cx, n_in, n_out)
    res = [g.create_sample_resource(synth((ch, 300 + 37 * i), 40 + i)) for i, ch in enumerate((2, 1))]
    for v in range(V):
        g.sampler_set_sample(smp, res[v % 2], True, voice=v)
        g.sampler_set_loop_range(smp, "full", voice=v)
        g.sampler_play(smp, voice=v)
    return cx, proc


def dag(G_in, G_out):
    """The generic lowering: a fused Volume -> Pan run and a Biquad and an SVF reading graph_in's ports (from the caller's rows when
    they are stream channels), a SumNode mixing them, graph_out ports fed by several nodes (fan-out), the rest unconnected."""
    def build(lib, n_in, n_out, V, bus, mcf=0):
        cx = ctx(lib, G_in, G_out, V, bus, mcf)
        g = cx.graph
        gin, gout = g.graph_in_node(), g.graph_out_node()
        vol, pn = g.add_node(2, 2, VolumeNode(100.0)), g.add_node(2, 2, PanNode(0.0))
        bq, sv = g.add_node(1, 1, BiquadNode(2)), g.add_node(1, 1, SvfNode(1))
        mix, clip = g.add_node(3, 1, SumNode()), g.add_node(1, 1, HardClipNode(-3.0))
        for c in range(2):
            if G_in:
                g.connect(gin, c % G_in, vol, c, False)
            g.connect(vol, c, pn, c, False)
        if G_in:
            g.connect(gin, G_in - 1, bq, 0, False)
            g.connect(gin, G_in - 1, sv, 0, False)
        g.connect(pn, 0, mix, 0, False); g.connect(bq, 0, mix, 1, False); g.connect(sv, 0, mix, 2, False)
        g.connect(mix, 0, clip, 0, False)
        for p, (src, sp) in enumerate([(clip, 0), (pn, 1), (bq, 0), (pn, 0), (sv, 0)]):
            if p < G_out:
                g.connect(src, sp, gout, p, False)
        g.set_percent_volume(vol, voice_pcts(V, 4))
        g.set_pan(pn, np.random.default_rng(5).uniform(-1, 1, V).astype(f32))
        g.set_biquad_coeffs(bq, np.array([design_rbj(lib, 0, 2000.0 + 500 * s, 0.9, 0.0, SR) for s in range(2)], f32))
        g.set_svf_coeffs(sv, np.array([design_svf(lib, 1, 900.0, 1.2, SR)], f32))
        return cx, activate(cx, n_in, n_out)
    return build


def plugin(lib, n_in, n_out, V, bus, mcf=0):
    """graph_in(2) -> the fir1 plugin (tests/plugins/fir1_plugin.cu) -> graph_out(2)"""
    cx = ctx(lib, 2, 2, V, bus, mcf)
    g = cx.graph
    cu = g.add_custom_node(2, 2, *pf.new_node(0.4, pf.RULE_ALL_IF_ALL_INPUTS))
    for c in range(2):
        g.connect(g.graph_in_node(), c, cu, c, False)
        g.connect(cu, c, g.graph_out_node(), c, False)
    return cx, activate(cx, n_in, n_out)


def inputs(V, n_in, T, seed):
    x = synth((V, n_in, T), seed)
    if V > 1 and n_in:
        x[V // 2] = 0.0  # a silent voice
    return x


# ---- entry points: one call -> (output, mask or None) --------------------------------------------------------------------------
def call_planar(proc, x, n_out, bus):
    V, n_in, T = x.shape
    out = np.full((n_out, T) if bus else (V, n_out, T), np.nan, f32)
    rc, mask = proc.process_planar(np.ascontiguousarray(x), out, n_in, n_out, T)
    assert rc == 0, (rc, proc._lib.last_device_error())
    return out, mask


def call_interleaved(proc, x, n_out, bus):
    V, n_in, T = x.shape
    out = np.full((1 if bus else V, T, n_out), np.nan, f32)
    rc = proc.process_interleaved(np.ascontiguousarray(x.transpose(0, 2, 1)), out, n_in, n_out, T)
    assert rc == 0, (rc, proc._lib.last_device_error())
    return out, None


def call_device(proc, x, n_out, bus):
    import torch
    V, n_in, T = x.shape
    d_in = torch.from_numpy(np.ascontiguousarray(x)).cuda()
    d_out = torch.full((n_out, T) if bus else (V, n_out, T), float("nan"), dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    rc = proc.process_planar_device(d_in.data_ptr(), d_out.data_ptr(), n_in, n_out, T)
    assert rc == 0 and proc.sync() == 0, (rc, proc._lib.last_device_error())
    return d_out.cpu().numpy(), None


ENTRIES = {"planar": call_planar, "interleaved": call_interleaved, "device": call_device}


def run(lib, build, n_in, n_out, V, bus, Ts, entry="planar", mcf=0):
    cx, proc = build(lib, n_in, n_out, V, bus, mcf)
    call = ENTRIES[entry]
    res = [call(proc, inputs(V, n_in, T, 10 + i), n_out, bus) for i, T in enumerate(Ts)]
    proc.free(); cx.update(); cx.free()
    return res


def compare(gpu, oracle, build, n_in, n_out, V, bus, Ts=(5 * F + 9, F, 3 * F), entry="planar", mcf=0):
    # the device entry point is compared against the oracle's planar one: the same layout
    got = run(gpu, build, n_in, n_out, V, bus, Ts, entry, mcf)
    want = run(oracle, build, n_in, n_out, V, bus, Ts, "planar" if entry == "device" else entry, mcf)
    for i, ((yg, mg), (yo, mo)) in enumerate(zip(got, want)):
        assert_bit_exact(yg, yo, f"call {i}")
        if mg is not None:
            assert mg == mo, f"call {i}: silence mask {mg:#x} != {mo:#x}"
    return got


# ============================== CPU: known answers of the oracle ==============================================================
def test_surplus_graph_in_port_is_a_live_zero(oracle):
    """S1: a mono Volume on graph_in port 1 of a mono stream reads +0.0, flagged silent by prepare_graph_inputs and then overwritten by
    graph_in's Dummy (schedule.rs:244-252,338-341): the Volume sees a live input, so graph_out's port is not flagged."""
    cx = ctx(oracle, 2, 1, 1, False)
    g = cx.graph
    vol = g.add_node(1, 1, VolumeNode(50.0))
    g.connect(g.graph_in_node(), 1, vol, 0, False)
    g.connect(vol, 0, g.graph_out_node(), 0, False)
    proc = activate(cx, 1, 1)
    y, m = call_planar(proc, synth((1, 1, 3 * F), 1), 1, False)
    assert not y.view(np.uint32).any() and m == 0
    proc.free(); cx.update(); cx.free()


@pytest.mark.parametrize("bus,V", [(False, 3), (True, 1), (True, 3)])
def test_surplus_outputs_are_positive_zero_and_never_flagged(oracle, bus, V):
    """S3 and S4: a 2-port graph_out on a 5-channel stream writes +0.0 to channels 2-4 and flags at most channels 0-1 (util.rs:96,
    schedule.rs:267-276); on a 1-channel stream it reads port 0 only, and the mask covers that one channel."""
    for muted in (False, True):
        y, m = run(oracle, gain_pan(muted=muted), 2, 5, V, bus, [2 * F])[0]
        live, surplus = (y[:2], y[2:]) if bus else (y[:, :2], y[:, 2:])
        assert not surplus.view(np.uint32).any() and m & ~0b11 == 0
        assert live.any() != muted
    assert run(oracle, gain_pan(muted=True), 2, 1, V, bus, [2 * F])[0][1] == 1


def test_all_muted_bus_with_surplus_channels_has_mask_zero(oracle):
    """With two or more voices the bus tree's SumNodes see 2 n_out inputs, and the surplus ones are never flagged (sum.rs:52-56): an
    all-muted stereo bus on a 6-channel stream has mask 0, on a 2-channel stream mask 0b11."""
    assert run(oracle, gain_pan(muted=True), 2, 6, 4, True, [2 * F])[0][1] == 0
    assert run(oracle, gain_pan(muted=True), 2, 2, 4, True, [2 * F])[0][1] == 0b11
    assert run(oracle, gain_pan(muted=True), 2, 6, 1, True, [2 * F])[0][1] == 0b11  # one voice: the root is the voice


@pytest.mark.parametrize("seed", range(8))
def test_oracle_equals_pyref_on_mismatched_interleaved(oracle, seed):
    """process_interleaved on random G_in / G_out / n_in / n_out, including n_out == 2 with G_out != 2 (no stereo fast path)"""
    rng = np.random.default_rng(300 + seed)
    G_in, G_out = int(rng.integers(1, 4)), int(rng.integers(1, 4))
    n_in, n_out = int(rng.integers(0, 5)), (2 if seed < 3 else int(rng.integers(1, 6)))
    cx = ctx(oracle, G_in, G_out, 1, False)
    g = cx.graph
    py = {int(g.graph_in_node()): pyref.Dummy(), int(g.graph_out_node()): pyref.Dummy()}
    vols = []
    for p in range(G_out):
        pct = float(rng.choice([0.0, 60.0, 100.0]))
        vol = g.add_node(1, 1, VolumeNode(pct)); py[int(vol)] = pyref.Volume(pct, SR, 16); vols.append(vol)
        g.connect(g.graph_in_node(), int(rng.integers(G_in)), vol, 0, False)
        g.connect(vol, 0, g.graph_out_node(), p, False)
    sched, nb = g.compile_internal(16)
    ex = pyref.Executor([(int(s.id), s.input_buffers, s.output_buffers) for s in sched], nb, 16, py)
    proc = activate(cx, n_in, n_out, 16)
    for call in range(3):
        T = int(rng.choice([16, 37]))
        x = np.ascontiguousarray(synth((T, n_in), 50 * seed + call))
        out = np.full((T, n_out), np.nan, f32)
        assert proc.process_interleaved(x, out, n_in, n_out, T) == 0
        want = ex.process_interleaved(x, n_out)
        assert np.array_equal(out.view(np.uint32), want.view(np.uint32)), (seed, call)
    proc.free(); cx.update(); cx.free()


# ============================== GPU: product == oracle =========================================================================
LAYOUTS = [(1, 2), (0, 2), (4, 2), (2, 1), (2, 6), (1, 8), (0, 6), (2, 2)]  # (n_in, n_out) around graph_in(2) / graph_out(2)


@pytest.mark.gpu
@pytest.mark.parametrize("bus", [False, True])
@pytest.mark.parametrize("V", [1, 2, 65])
@pytest.mark.parametrize("n_in,n_out", LAYOUTS)
def test_fused_chain(gpu, oracle, n_in, n_out, V, bus):
    compare(gpu, oracle, gain_pan(), n_in, n_out, V, bus)


@pytest.mark.gpu
@pytest.mark.parametrize("G_in,G_out,n_in,n_out", [(2, 2, 1, 6), (1, 1, 2, 8), (2, 1, 0, 2), (1, 2, 4, 1)])
@pytest.mark.parametrize("V,bus", [(1100, True), (1100, False), (64, True)])
def test_fused_chain_many_voices(gpu, oracle, G_in, G_out, n_in, n_out, V, bus):
    compare(gpu, oracle, gain_pan(G_in, G_out), n_in, n_out, V, bus, Ts=(3 * F + 5, F))


@pytest.mark.gpu
@pytest.mark.parametrize("V,bus", [(1, False), (65, True), (2, True)])
def test_sampler_chain_on_six_channels(gpu, oracle, V, bus):
    compare(gpu, oracle, sampler_chain, 0, 6, V, bus)


@pytest.mark.gpu
@pytest.mark.parametrize("bus", [False, True])
@pytest.mark.parametrize("V", [2, 65])
@pytest.mark.parametrize("G_in,G_out,n_in,n_out", [(3, 6, 1, 2), (3, 2, 2, 6), (2, 1, 4, 8), (1, 6, 0, 1), (0, 2, 2, 2), (3, 6, 3, 8),
                                                   (2, 6, 2, 2), (3, 1, 2, 6)])
def test_generic_lowering(gpu, oracle, G_in, G_out, n_in, n_out, V, bus):
    compare(gpu, oracle, dag(G_in, G_out), n_in, n_out, V, bus)


@pytest.mark.gpu
@pytest.mark.parametrize("n_in,n_out,V,bus", [(1, 2, 3, False), (0, 6, 65, True), (4, 1, 2, False)])
def test_plugin_fed_a_surplus_port(gpu, oracle, n_in, n_out, V, bus):
    compare(gpu, oracle, plugin, n_in, n_out, V, bus)


@pytest.mark.gpu
@pytest.mark.parametrize("entry", ["interleaved", "device"])
@pytest.mark.parametrize("build,n_in,n_out,V,bus", [(gain_pan(1, 1), 1, 2, 1, False), (gain_pan(2, 3), 2, 2, 3, False), (gain_pan(), 1, 6, 65, True),
                                                    (dag(3, 6), 2, 2, 2, True), (dag(3, 1), 1, 2, 2, False), (gain_pan(muted=True), 2, 6, 3, True)])
def test_entry_points(gpu, oracle, entry, build, n_in, n_out, V, bus):
    """n_out == 2 with G_out != 2 interleaves channel by channel (processor.rs:122-133)"""
    compare(gpu, oracle, build, n_in, n_out, V, bus, entry=entry)


@pytest.mark.gpu
@pytest.mark.parametrize("build,n_in,n_out,bus", [(gain_pan(), 1, 6, True), (gain_pan(), 0, 6, False), (dag(3, 6), 1, 2, True)])
def test_chunked_and_block_sized_calls_replay(gpu, oracle, build, n_in, n_out, bus):
    """calls of 5 blocks against a 2-block reserve, then block-sized calls, whose steady chunks replay as CUDA graphs"""
    V = 9
    Ts = (5 * F + 9,) + (F,) * 6
    compare(gpu, oracle, build, n_in, n_out, V, bus, Ts=Ts, mcf=2 * F)
    cx, proc = build(gpu, n_in, n_out, V, bus, 2 * F)
    x = inputs(V, n_in, F, 1)
    replays = []
    for _ in range(5):
        call_planar(proc, x, n_out, bus)
        replays.append(proc.graph_replays())
    proc.free(); cx.update(); cx.free()
    assert replays[1] >= 1 and replays[4] - replays[1] == 3, replays


@pytest.mark.gpu
def test_bus_width_is_the_live_width(gpu, oracle):
    """a bus is refused only when its live width min(G_out, n_out) exceeds 8"""
    compare(gpu, oracle, dag(2, 9), 2, 2, 3, True)
    compare(gpu, oracle, surround(8), 8, 12, 3, True)


def surround(C):
    def build(lib, n_in, n_out, V, bus, mcf=0):
        cx = ctx(lib, C, C, V, bus, mcf)
        g = cx.graph
        for z in range(0, C, 2):
            vol = g.add_node(2, 2, VolumeNode(100.0))
            for c in range(2):
                g.connect(g.graph_in_node(), z + c, vol, c, False)
                g.connect(vol, c, g.graph_out_node(), z + c, False)
            g.set_percent_volume(vol, voice_pcts(V, z))
        return cx, activate(cx, n_in, n_out)
    return build


@pytest.mark.gpu
def test_graph_out_port_count_change_while_active(gpu, oracle):
    """set_num_inputs on graph_out while the stream runs (graph.rs:349): the next update swaps in the new schedule, which the
    device lowers again, and the stream keeps playing"""
    V, n_in, n_out = 5, 2, 4
    outs = []
    for lib in (gpu, oracle):
        cx, proc = gain_pan()(lib, n_in, n_out, V, False)
        g = cx.graph
        res = [call_planar(proc, inputs(V, n_in, 2 * F, 1), n_out, False)]
        g.set_num_inputs(g.graph_out_node(), 3)
        st = cx.update()
        assert st.graph_error is None, (st, cx.last_error())
        res += [call_planar(proc, inputs(V, n_in, 2 * F, 2 + i), n_out, False) for i in range(2)]
        g.set_num_inputs(g.graph_out_node(), 1)
        assert cx.update().graph_error is None
        res += [call_planar(proc, inputs(V, n_in, 2 * F, 4 + i), n_out, False) for i in range(2)]
        proc.free(); cx.update(); cx.free()
        outs.append(res)
    for i, ((yg, mg), (yo, mo)) in enumerate(zip(*outs)):
        assert_bit_exact(yg, yo, f"call {i}")
        assert mg == mo


@pytest.mark.gpu
def test_pull_stream_on_six_channels_with_graph_in_ports(gpu, oracle):
    """fw_stream_open renders with n_in = 0 (firewheel-cpal, lib.rs:177-178): a graph with graph_in ports reads zeros there, and a
    stereo graph on a 6-channel device plays on channels 0-1"""
    import time
    V, period, n_periods = 9, 192, 6
    build = dag(2, 2)
    cx, proc = build(gpu, 0, 6, V, True)
    st = proc.open_stream(6, SR, period, ring_periods=4)
    assert st is not None, gpu.last_device_error()
    got, t0 = [], time.time()
    while len(got) < n_periods:
        if st.frames_ready() >= period:
            y, k, status, _ = st.pull(period)
            assert k == period and status == 0
            got.append(y)
        else:
            assert time.time() - t0 < 60, "the producer made no progress"
            time.sleep(0.001)
    st.close()
    proc.free(); cx.update(); cx.free()
    cx, proc = build(oracle, 0, 6, V, True)
    want = []
    for _ in range(n_periods):
        out = np.full((period, 6), np.nan, f32)
        assert proc.process_interleaved(np.zeros(0, f32), out, 0, 6, period) == 0
        want.append(out)
    proc.free(); cx.update(); cx.free()
    assert_bit_exact(np.concatenate(got), np.concatenate(want), "pulled")


# launches per chunk (first call, steady call) of 4-block calls in one chunk: control + the data plane + one zero_rows launch when the
# stream has more output channels than graph_out has ports
LAUNCH_SHAPES = {
    "chain_matched": (gain_pan(), 2, 2, 37, False, (2, 2)),
    "chain_mono_in": (gain_pan(), 1, 2, 37, False, (2, 2)),
    "chain_no_in": (gain_pan(), 0, 2, 37, False, (2, 2)),
    "chain_six_out": (gain_pan(), 2, 6, 37, False, (3, 3)),
    "chain_mono_out": (gain_pan(), 2, 1, 37, False, (2, 2)),
    "chain_bus_six_out": (gain_pan(), 2, 6, 1024, True, (4, 4)),  # 16 partial buses: one combine level
    "chain_bus_mono_in": (gain_pan(), 1, 2, 1024, True, (3, 3)),
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(LAUNCH_SHAPES))
def test_launches_per_chunk(gpu, name):
    build, n_in, n_out, V, bus, expected = LAUNCH_SHAPES[name]
    cx, proc = build(gpu, n_in, n_out, V, bus)
    x = inputs(V, n_in, 4 * F, 5)
    deltas = []
    for _ in range(3):
        l0 = proc.kernel_launches()
        call_planar(proc, x, n_out, bus)
        deltas.append(proc.kernel_launches() - l0)
    replays = proc.graph_replays()
    proc.free(); cx.update(); cx.free()
    assert (deltas[0], deltas[2]) == expected, deltas
    assert replays == 2


# ---- two ranks: the live channels cross NCCL, the zero rows stay local -----------------------------------------------------------
@pytest.mark.gpu
def test_stereo_bus_on_six_channels_across_two_ranks(gpu):
    if gpu.device_count() < 2:
        pytest.skip("needs at least 2 GPUs")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
                        "--master-port", "29789", str(Path(__file__).resolve())], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    assert "channel layouts multigpu parity OK" in r.stdout


def _rank_main():
    """one rank: this rank's voices of a stereo bus on a 6-channel stream, against the oracle's tree of the per-rank trees"""
    import firewheel_b200 as fw
    import pyoracle
    from firewheel_b200 import rendezvous
    from sharding import tree_sum, voice_range
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    gpu, oracle = fw.load(), pyoracle.load()
    V, n_in, n_out, T = 201, 1, 6, 4 * F
    pct = voice_pcts(V, 9)
    x = synth((V, n_in, T), 31)

    def build(lib, a, b, device=0):
        cx = FirewheelGraphCtx(lib, AudioGraphConfig(num_graph_inputs=2, num_graph_outputs=2, num_voices=b - a, master_bus=True, device=device))
        g = cx.graph
        vol = g.add_node(2, 2, VolumeNode(100.0))
        for c in range(2):
            g.connect(g.graph_in_node(), c, vol, c, False); g.connect(vol, c, g.graph_out_node(), c, False)
        g.set_percent_volume(vol, pct[a:b])
        return cx, activate(cx, n_in, n_out)
    lo, hi = voice_range(V, rank, world)
    cx, proc = build(gpu, lo, hi, device=local)
    rendezvous.init_comm(gpu, proc, rank, world)
    out = np.full((n_out, T), np.nan, f32)
    for _ in range(2):
        rc, _ = proc.process_planar(np.ascontiguousarray(x[lo:hi]), out, n_in, n_out, T)
        assert rc == 0, (rc, gpu.last_device_error())
    parts = []
    for r in range(world):
        a, b = voice_range(V, r, world)
        ocx, oproc = build(oracle, a, b)
        y = np.zeros((n_out, T), f32)
        for _ in range(2):
            oproc.process_planar(np.ascontiguousarray(x[a:b]), y, n_in, n_out, T)
        parts.append(y.copy())
        oproc.free(); ocx.update(); ocx.free()
    ok = np.array_equal(out.view(np.uint32), tree_sum(parts).view(np.uint32))
    all_ok = bool(proc.comm_allgather(np.array([1 if ok else 0], np.int64)).min() == 1)
    proc.comm_allgather(np.zeros(1, np.int64))  # barrier: nobody tears its mailbox down while a peer still runs
    proc.free(); cx.update(); cx.free()
    rendezvous.cleanup(rank)
    if rank == 0:
        print("channel layouts multigpu parity", "OK" if all_ok else "MISMATCH")
    sys.exit(0 if all_ok else 1)


if __name__ == "__main__":
    _rank_main()
