"""Kernel launches per call, pinned for the shapes whose lowering decides how many launches a call costs: fused chain stages, fused
runs of the generic lowering (DESIGN.md §4), runs that read the caller's rows, per-channel pointwise nodes with their silence fix, and
the odd tail of two-channels-per-launch copies. Outputs stay bit-exact when a run is split into more launches, so only the count
shows it. Each call carries no pending parameter command (every store would add a launch); the first call is launched kernel by
kernel, the third replays the CUDA graph captured by the second where the plan allows it."""
import pytest

from conftest import synth
from firewheel_b200 import (AudioGraphConfig, BiquadNode, DelayNode, FirewheelGraphCtx, HardClipNode, MonoToStereoNode, PanNode, StereoToMonoNode,
                            SumNode, SvfNode, VolumeNode)
from helpers import SR, chain, run_planar

pytestmark = pytest.mark.gpu

F = 128


def generic(lib, n_in, n_out, V, bus, wire):
    """A voice graph built by wire(g, gin, gout); it is no port-to-port chain, so it takes the generic lowering."""
    cx = FirewheelGraphCtx(lib, AudioGraphConfig(num_graph_inputs=n_in, num_graph_outputs=n_out, num_voices=V, master_bus=bus))
    g = cx.graph
    wire(g, g.graph_in_node(), g.graph_out_node())
    proc = cx.activate(SR, n_in, n_out, F)
    assert proc is not None
    st = cx.update()
    assert st.kind == "Active" and st.graph_error is None, (st, cx.last_error())
    return cx, proc


def gain_pan_bus(lib):  # 1100 voices: 18 partial buses, two combine levels
    cx, proc, _ = chain(lib, 2, [(lambda: VolumeNode(80.0), 2, 2), (lambda: PanNode(0.3), 2, 2)], voices=1100, master_bus=True, max_block=F)
    return cx, proc, 2, 2, 1100, True


def biquad_delay_volume(lib):
    nodes = [(lambda: BiquadNode(2), 2, 2), (lambda: DelayNode(100), 2, 2), (lambda: VolumeNode(70.0), 2, 2)]
    cx, proc, _ = chain(lib, 2, nodes, voices=37, max_block=F)
    return cx, proc, 2, 2, 37, False


def dag(lib):  # the benchmark's dag voice graph
    def wire(g, gin, gout):
        dry, svf, wet1 = g.add_node(2, 2, VolumeNode(80.0)), g.add_node(2, 2, SvfNode(2)), g.add_node(2, 2, VolumeNode(40.0))
        bq, wet2 = g.add_node(2, 2, BiquadNode(2)), g.add_node(2, 2, VolumeNode(30.0))
        mix, pn = g.add_node(6, 2, SumNode()), g.add_node(2, 2, PanNode(0.0))
        for c in range(2):
            g.connect(gin, c, dry, c, False); g.connect(gin, c, svf, c, False); g.connect(gin, c, bq, c, False)
            g.connect(svf, c, wet1, c, False); g.connect(bq, c, wet2, c, False)
            g.connect(dry, c, mix, c, False); g.connect(wet1, c, mix, 2 + c, False); g.connect(wet2, c, mix, 4 + c, False)
            g.connect(mix, c, pn, c, False); g.connect(pn, c, gout, c, False)
    return (*generic(lib, 2, 2, 64, True, wire), 2, 2, 64, True)


def swapped_run(bus):
    def build(lib):  # gain -> pan read graph_in's channels (1, 0) and ride in graph_out: no pool copy of the inputs
        def wire(g, gin, gout):
            vol, pn = g.add_node(2, 2, VolumeNode(80.0)), g.add_node(2, 2, PanNode(-0.4))
            for c in range(2):
                g.connect(gin, 1 - c, vol, c, False); g.connect(vol, c, pn, c, False); g.connect(pn, c, gout, c, False)
        return (*generic(lib, 2, 2, 37, bus, wire), 2, 2, 37, bus)
    return build


def mono_volume_clip(lib):  # one channel each: per-channel launches, then the silence fix
    def wire(g, gin, gout):
        vol, clip = g.add_node(1, 1, VolumeNode(80.0)), g.add_node(1, 1, HardClipNode(-6.0))
        g.connect(gin, 0, vol, 0, False); g.connect(gin, 0, clip, 0, False)
        g.connect(vol, 0, gout, 0, False); g.connect(clip, 0, gout, 1, False)
    return (*generic(lib, 1, 2, 37, False, wire), 1, 2, 37, False)


def m2s_s2m(lib):
    def wire(g, gin, gout):
        s2m, m2s = g.add_node(2, 1, StereoToMonoNode()), g.add_node(1, 2, MonoToStereoNode())
        for c in range(2):
            g.connect(gin, c, s2m, c, False); g.connect(m2s, c, gout, 1 - c, False)
        g.connect(s2m, 0, m2s, 0, False)
    return (*generic(lib, 2, 2, 37, False, wire), 2, 2, 37, False)


def sum_copy(lib):  # a 1-port SumNode is a copy
    def wire(g, gin, gout):
        s = g.add_node(2, 2, SumNode())
        for c in range(2):
            g.connect(gin, c, s, c, False); g.connect(s, c, gout, 1 - c, False)
    return (*generic(lib, 2, 2, 37, False, wire), 2, 2, 37, False)


def copy3(lib):  # three channels: graph_in and graph_out copies and the clip each end in a one-channel launch
    def wire(g, gin, gout):
        clip = g.add_node(3, 3, HardClipNode(-3.0))
        for c in range(3):
            g.connect(gin, c, clip, c, False); g.connect(clip, c, gout, c, False)
    return (*generic(lib, 3, 3, 37, False, wire), 3, 3, 37, False)


SHAPES = {
    "gain_pan_bus": gain_pan_bus,
    "biquad_delay_volume": biquad_delay_volume,
    "dag": dag,
    "swapped_run": swapped_run(False),
    "swapped_run_bus": swapped_run(True),
    "mono_volume_clip": mono_volume_clip,
    "m2s_s2m": m2s_s2m,
    "sum_copy": sum_copy,
    "copy3": copy3,
}

# (first call, steady call)
EXPECTED = {
    "gain_pan_bus": (4, 4),
    "biquad_delay_volume": (3, 3),
    "dag": (9, 9),
    "swapped_run": (2, 2),
    "swapped_run_bus": (2, 2),
    "mono_volume_clip": (7, 7),
    "m2s_s2m": (8, 8),
    "sum_copy": (4, 4),
    "copy3": (10, 10),
}


def launches_per_call(lib, name):
    cx, proc, n_in, n_out, V, bus = SHAPES[name](lib)
    x = synth((V, n_in, 4 * F), 5)
    deltas = []
    for _ in range(3):
        l0 = proc.kernel_launches()
        run_planar(proc, x, n_out, bus)
        deltas.append(proc.kernel_launches() - l0)
    proc.free(); cx.update(); cx.free()
    return deltas[0], deltas[2]


@pytest.mark.parametrize("name", sorted(SHAPES))
def test_launches_per_call(gpu, name):
    assert launches_per_call(gpu, name) == EXPECTED[name]
