"""Kernel launches per call of the fused chain's stage splits (DESIGN.md §4): which nodes share a stage, which stages ping-pong through
the two scratch buffers, and when a copy stage is forced in front of the master bus. Outputs stay bit-exact when a chain is split into
more stages, so only the count shows it. The first call is launched kernel by kernel; the third replays the CUDA graph captured by the
second where the plan allows it (a delay or reverb keeps it on plain launches)."""
import pytest

from conftest import synth
from firewheel_b200 import (AudioGraphConfig, BiquadNode, ConvReverbNode, DelayNode, FirewheelGraphCtx, MonoToStereoNode, PanNode, SamplerNode,
                            SvfNode, VolumeNode)
from helpers import SR, chain, run_planar

pytestmark = pytest.mark.gpu

F = 128


def fused_chain(n_ch, nodes, V=37):
    def build(lib):
        cx, proc, _ = chain(lib, n_ch, nodes, voices=V, max_block=F)
        return cx, proc, n_ch, nodes[-1][2], V, False
    return build


def reverb_ir():
    return synth((2, 64), 11) * 0.1


def sampler_chain_bus(lib):  # config 5's shape: sampler head, both scratch buffers, and the copy stage that feeds the bus after the reverb
    cx = FirewheelGraphCtx(lib, AudioGraphConfig(num_graph_inputs=0, num_graph_outputs=2, num_voices=70, master_bus=True))
    g = cx.graph
    prev = g.add_node(0, 2, SamplerNode(100.0))
    for node in (VolumeNode(80.0), PanNode(0.2), BiquadNode(2), ConvReverbNode(reverb_ir())):
        nid = g.add_node(2, 2, node)
        for c in range(2):
            g.connect(prev, c, nid, c, False)
        prev = nid
    for c in range(2):
        g.connect(prev, c, g.graph_out_node(), c, False)
    proc = cx.activate(SR, 0, 2, F)
    assert proc is not None
    st = cx.update()
    assert st.kind == "Active" and st.graph_error is None, (st, cx.last_error())
    return cx, proc, 0, 2, 70, True


# name: (builder, (first call, steady call))
SHAPES = {
    "reverb_only": (fused_chain(2, [(lambda: ConvReverbNode(reverb_ir()), 2, 2)]), (3, 3)),  # config 4's shape
    "sampler_chain_bus": (sampler_chain_bus, (8, 8)),
    "svf_delay": (fused_chain(2, [(lambda: SvfNode(2), 2, 2), (lambda: DelayNode(100), 2, 2)]), (3, 3)),  # a delay joins biquad passes only
    "lone_delay": (fused_chain(2, [(lambda: DelayNode(100), 2, 2)]), (2, 2)),
    "biquad_volume_svf_delay": (fused_chain(2, [(lambda: BiquadNode(2), 2, 2), (lambda: VolumeNode(70.0), 2, 2), (lambda: SvfNode(2), 2, 2),
                                                (lambda: DelayNode(100), 2, 2)]), (5, 5)),  # four stages through both scratch buffers
    "mono_m2s_stereo": (fused_chain(1, [(lambda: VolumeNode(70.0), 1, 1), (lambda: MonoToStereoNode(), 1, 2), (lambda: BiquadNode(2), 2, 2)]), (3, 3)),
}


@pytest.mark.parametrize("name", sorted(SHAPES))
def test_chain_launches_per_call(gpu, name):
    build, expected = SHAPES[name]
    cx, proc, n_in, n_out, V, bus = build(gpu)
    x = synth((V, n_in, 4 * F), 5)
    deltas = []
    for _ in range(3):
        l0 = proc.kernel_launches()
        run_planar(proc, x, n_out, bus)
        deltas.append(proc.kernel_launches() - l0)
    proc.free(); cx.update(); cx.free()
    assert (deltas[0], deltas[2]) == expected
