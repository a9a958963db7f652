"""Processor lifecycle on the device: an activation that fails part-way releases what it had built, and the process goes on working."""
import numpy as np
import pytest

from conftest import synth
from firewheel_b200 import AudioGraphConfig, FirewheelGraphCtx, PanNode, VolumeNode
from helpers import SR, assert_bit_exact, chain, f32, run_planar

pytestmark = pytest.mark.gpu


def test_failed_activation_then_fresh_context(gpu, oracle):
    V, F = 64, 256
    # I/O staging for 64 stereo voices of 2^28 frames is 128 GiB per direction: cudaMalloc refuses it with an ordinary API error,
    # after the stream, the events, the pinned buffers and the bus-sized output staging were created
    cx = FirewheelGraphCtx(gpu, AudioGraphConfig(num_graph_inputs=2, num_graph_outputs=2, num_voices=V, master_bus=True, max_call_frames=1 << 28))
    with pytest.raises(RuntimeError, match=r"device allocation failed \(I/O staging"):
        cx.activate(SR, 2, 2, F)
    assert not cx.is_activated()
    cx.free()

    # the same process: a fresh gain -> pan -> bus context is bit-exact against the oracle, through the planar entry point and through
    # the interleaved one, whose (de)interleave launches check the runtime's pending error
    rng = np.random.default_rng(11)
    pct = rng.uniform(25, 100, V).astype(f32)
    pan = rng.uniform(-1, 1, V).astype(f32)
    T = F * 4
    x = synth((V, 2, T), 11)
    xi = np.ascontiguousarray(synth((V, 2, T), 12).transpose(0, 2, 1))  # [voice][frame][channel]

    def setup(cx, ids):
        cx.graph.set_percent_volume(ids[0], pct)
        cx.graph.set_pan(ids[1], pan)

    outs = []
    for lib in (gpu, oracle):
        cx, proc, _ = chain(lib, 2, [(lambda: VolumeNode(100.0), 2, 2), (lambda: PanNode(0.0), 2, 2)], voices=V, master_bus=True,
                            max_block=F, setup=setup)
        planar, mask = run_planar(proc, x, 2, master_bus=True)
        inter = np.full((T, 2), np.nan, dtype=f32)
        rc = proc.process_interleaved(xi, inter, 2, 2, T)
        assert rc == 0, (rc, lib.last_device_error())
        outs.append((planar, mask, inter))
        proc.free()
        cx.update()
        cx.free()
    (yg, mg, ig), (yo, mo, io) = outs
    assert_bit_exact(yg, yo, "planar gain -> pan -> bus after a failed activation")
    assert mg == mo
    assert_bit_exact(ig, io, "interleaved gain -> pan -> bus after a failed activation")
