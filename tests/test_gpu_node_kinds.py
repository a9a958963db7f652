"""Per-kind facts of the node-kind table (graph.cpp kNodeKinds) that outputs and launch counts do not show:
- every kind with per-channel device state is activated again when a live node's port count changes (test_gpu_timed_events.py
  covers the BiquadNode);
- a plan replays its steady calls from a CUDA graph unless a node's kernel arguments change from call to call. A replayable plan kept
  on plain launches gives the same outputs and launch counts, only slower, so the replays of the steady call are pinned for every
  shape of the launch-count tests."""
import numpy as np
import pytest

import test_gpu_chain_launch_counts as chain_counts
import test_gpu_launch_counts as launch_counts
from conftest import synth
from helpers import SR, assert_bit_exact, run_planar

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("kind", ["svf", "delay", "conv_reverb"])
def test_port_count_change_reactivates_every_kind_with_per_channel_state(gpu, kind):
    """set_num_inputs / set_num_outputs on an activated node (graph.rs:315-393): its per-channel device state no longer fits, so the
    node is activated again with the new counts (fresh state) instead of running out of bounds. The delay line is several blocks long,
    so its ring carries samples from call to call."""
    from firewheel_b200 import AudioGraphConfig, ConvReverbNode, DelayNode, FirewheelGraphCtx, SvfNode, design_svf
    V, F = 6, 64
    x = synth((V, 4, 4 * F), 8)

    def add(g, ports):
        if kind == "svf":
            node = g.add_node(ports, ports, SvfNode(1))
            g.set_svf_coeffs(node, np.stack([[design_svf(gpu, 0, 1000.0 + 100 * v, 0.8, SR)] for v in range(V)]).astype(np.float32))
            return node
        if kind == "delay":
            return g.add_node(ports, ports, DelayNode(3 * F + 17))
        return g.add_node(ports, ports, ConvReverbNode(synth((4, 96), 9) * 0.1))

    def build(ports):
        cx = FirewheelGraphCtx(gpu, AudioGraphConfig(num_graph_inputs=4, num_graph_outputs=4, num_voices=V))
        g = cx.graph
        node = add(g, ports)
        for c in range(4):
            if c < ports:
                g.connect(g.graph_in_node(), c, node, c, False); g.connect(node, c, g.graph_out_node(), c, False)
            else:
                g.connect(g.graph_in_node(), c, g.graph_out_node(), c, False)
        proc = cx.activate(SR, 4, 4, F)
        assert cx.update().graph_error is None, cx.last_error()
        return cx, proc, node
    cx, proc, node = build(2)
    run_planar(proc, x, 4)
    g = cx.graph
    for c in (2, 3):
        assert g.disconnect(g.graph_in_node(), c, g.graph_out_node(), c)
    g.set_num_inputs(node, 4); g.set_num_outputs(node, 4)
    for c in (2, 3):
        g.connect(g.graph_in_node(), c, node, c, False); g.connect(node, c, g.graph_out_node(), c, False)
    assert cx.update().graph_error is None, cx.last_error()
    run_planar(proc, x, 4)          # Q11: the first block after the swap reads zero inputs
    y_live, _ = run_planar(proc, x, 4)
    proc.free(); cx.update(); cx.free()
    cx2, proc2, _ = build(4)
    run_planar(proc2, np.concatenate([np.zeros((V, 4, F), np.float32), x[:, :, F:]], axis=2), 4)   # what the re-activated node saw in the swap call
    y_fresh, _ = run_planar(proc2, x, 4)
    proc2.free(); cx2.update(); cx2.free()
    assert_bit_exact(y_live, y_fresh, f"re-activated 4-channel {kind}")


# graph replays of the steady (third) call: 0 where a delay or a reverb keeps the plan on plain launches
BUILDERS = {**launch_counts.SHAPES, **{name: s[0] for name, s in chain_counts.SHAPES.items()}}
REPLAYS = {
    "gain_pan_bus": 1, "biquad_delay_volume": 0, "dag": 1, "swapped_run": 1, "swapped_run_bus": 1, "mono_volume_clip": 1, "m2s_s2m": 1,
    "sum_copy": 1, "copy3": 1,
    "reverb_only": 0, "sampler_chain_bus": 0, "svf_delay": 0, "lone_delay": 0, "biquad_volume_svf_delay": 0, "mono_m2s_stereo": 1,
}
assert set(REPLAYS) == set(BUILDERS), "every launch-count shape has its steady-call replays pinned"


@pytest.mark.parametrize("name", sorted(REPLAYS))
def test_steady_call_replays_unless_a_node_varies_from_call_to_call(gpu, name):
    cx, proc, n_in, n_out, V, bus = BUILDERS[name](gpu)
    x = synth((V, n_in, 4 * launch_counts.F), 5)
    for _ in range(2):
        run_planar(proc, x, n_out, bus)
    r0 = proc.graph_replays()
    run_planar(proc, x, n_out, bus)
    replays = proc.graph_replays() - r0
    proc.free(); cx.update(); cx.free()
    assert replays == REPLAYS[name]
