"""The host-buffer entry points (process_planar, process_interleaved) and the device-buffer one (process_planar_device + sync) on the
two outcomes of a call that every entry point must report the same way:

* a processor dropped mid-call (Stop queued by the context): return FW_PROC_DROP_PROCESSOR, every output sample +0.0 (the host chunk
  the device ran as well as the rest of the caller's buffer, filled on the host) and no silence mask;
* an error the control kernel writes into the plan's error word (the record-budget overflow of DESIGN §5: a gain ramp that stays a
  transient for more blocks than the record buffers hold): return FW_PROC_DEVICE_ERROR for the call that overflowed, and 0 for the
  next call on the same processor (the error is not sticky)."""
import ctypes as C
import math

import numpy as np
import pytest

from conftest import synth
from firewheel_b200 import AudioGraphConfig, FirewheelGraphCtx, VolumeNode
from firewheel_b200._capi import PROC_DEVICE_ERROR, PROC_DROP_PROCESSOR

pytestmark = pytest.mark.gpu

SR = 48000
f32 = np.float32


def volume_ctx(lib, V, F, max_call_frames, pct, bus=False):
    """graph_in(2) -> VolumeNode(pct) -> graph_out(2), activated and compiled. The volume starts un-smoothed at `pct`."""
    cx = FirewheelGraphCtx(lib, AudioGraphConfig(num_graph_inputs=2, num_graph_outputs=2, num_voices=V, master_bus=bus, max_call_frames=max_call_frames))
    g = cx.graph
    vol = g.add_node(2, 2, VolumeNode(pct))
    for c in range(2):
        g.connect(g.graph_in_node(), c, vol, c, False)
        g.connect(vol, c, g.graph_out_node(), c, False)
    proc = cx.activate(SR, 2, 2, F)
    st = cx.update()
    assert st.kind == "Active" and st.graph_error is None, (st, cx.last_error())
    return cx, proc, vol


# ---- drop -----------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("bus", [False, True])
@pytest.mark.parametrize("entry", ["planar", "interleaved"])
def test_drop_zeroes_the_whole_call(gpu, entry, bus):
    """deactivate(stream_is_running=1) without a stream thread times out (about 3 s) and leaves Stop queued for the processor. The next
    call, 7.5 blocks against a 3-block reserve, sees Stop at its first chunk: the first host chunk is silenced on the device and staged
    out, the remaining 4.5 blocks are zeroed on the host."""
    V, F = 3, 64
    T = 7 * F + F // 2
    cx, proc, _ = volume_ctx(gpu, V, F, 3 * F, 100.0, bus)
    cx.deactivate(1)
    Vo = 1 if bus else V
    x = synth((V, 2, T), 11)
    if entry == "planar":
        out = np.full((Vo, 2, T), np.nan, dtype=f32)
        mask = C.c_uint64(0xdeadbeef)
        rc = gpu.processor_process_planar(proc._h, x.ctypes.data, out.ctypes.data, 2, 2, T, 0.0, 0, C.byref(mask))
        assert mask.value == 0
    else:
        xi = np.ascontiguousarray(x.transpose(0, 2, 1))  # [voice][frame][channel]
        out = np.full((Vo, T, 2), np.nan, dtype=f32)
        rc = proc.process_interleaved(xi, out, 2, 2, T)
    assert rc == PROC_DROP_PROCESSOR, (rc, gpu.last_device_error())
    bits = out.view(np.uint32)
    first = bits[:, :, :3 * F] if entry == "planar" else bits[:, :3 * F, :]
    rest = bits[:, :, 3 * F:] if entry == "planar" else bits[:, 3 * F:, :]
    assert not first.any(), "the device-run host chunk is not all +0.0"
    assert not rest.any(), "the host-filled rest of the call is not all +0.0"
    proc.free()
    cx.free()


# ---- record-budget overflow ---------------------------------------------------------------------------------------------------

def kt_max(F, max_call_frames, n_smoothers, n_samplers=0):
    """Record slots per voice and chunk, as alloc_plan (runtime.cu) sizes them."""
    tau = 0.01 * SR
    ramp_blocks = math.ceil(20.8 * tau / F) + 4
    kc = (max_call_frames + F - 1) // F + 1
    k = (ramp_blocks if n_smoothers else 4) + 8 * n_samplers
    return max(2, min(k, kc))


def transient_blocks(start, target, F, n_blocks):
    """Blocks, from the first, in which the gain smoother (kernels.cu: sm_set_and_process, f32 with no contraction) changes state
    after the target jumps from `start` to `target` at block 0 of a call on non-silent input. Every such block takes a record slot."""
    b = f32(np.exp(f32(-1.0) / (f32(10.0 / 1000.0) * f32(SR))))
    a = f32(f32(1.0) - b)
    eps = f32(0.00001)
    inp, last = f32(target), f32(start)
    t = f32(inp * a)
    for k in range(n_blocks):
        y0 = f32(t + f32(last * b))
        if abs(f32(inp - y0)) < eps:
            return k + 1          # the block that settles still changes the state (Active -> Deactivating)
        if y0 == last:
            return k              # f32 fixed point outside epsilon: a constant block, no state change
        y = y0
        for _ in range(1, F):
            y = f32(t + f32(y * b))
        last = y
    return n_blocks


@pytest.mark.parametrize("entry", ["planar", "interleaved", "device"])
def test_record_budget_overflow_is_reported_once(gpu, entry):
    """A downward gain jump from 10^6 % to 10^-3 % (raw gain 10^8 -> 10^-10) ramps for longer than the record buffers of one chunk
    hold. An upward jump would not do: it stops early at the f32 fixed point (Q10)."""
    V, F, K = 2, 256, 64
    mcf, T = K * F, K * F
    hi, lo = 1e6, 1e-3
    def raw_gain(pct):  # volume.rs:16-24 in f32
        n = f32(f32(pct) * f32(1.0 / 100.0))
        return f32(n * n)

    budget = kt_max(F, mcf, n_smoothers=1)
    ramp = transient_blocks(raw_gain(hi), raw_gain(lo), F, K)
    assert budget < ramp <= K, (budget, ramp)  # the call is one chunk and the ramp outlasts its record budget inside it
    cx, proc, vol = volume_ctx(gpu, V, F, mcf, hi)
    cx.graph.set_percent_volume(vol, lo)

    def call(frames):
        x = synth((V, 2, frames), frames)
        if entry == "planar":
            out = np.full((V, 2, frames), np.nan, dtype=f32)
            rc, _ = proc.process_planar(x, out, 2, 2, frames)
            return rc
        if entry == "interleaved":
            out = np.full((V, frames, 2), np.nan, dtype=f32)
            return proc.process_interleaved(np.ascontiguousarray(x.transpose(0, 2, 1)), out, 2, 2, frames)
        import torch
        d_in = torch.from_numpy(x).cuda()
        d_out = torch.empty((V, 2, frames), dtype=torch.float32, device="cuda")
        torch.cuda.synchronize()
        rc = proc.process_planar_device(d_in.data_ptr(), d_out.data_ptr(), 2, 2, frames)
        assert rc == 0, (rc, gpu.last_device_error())
        return PROC_DEVICE_ERROR if proc.sync() != 0 else 0

    assert call(T) == PROC_DEVICE_ERROR
    assert b"transient-block budget" in gpu.last_device_error()
    assert call(F) == 0, gpu.last_device_error()  # kt_max >= 2: one block cannot overflow
    proc.free()
    cx.update()
    cx.free()
