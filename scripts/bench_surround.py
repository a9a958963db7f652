"""Surround master bus on one GPU: 1024 voices of graph_in(C) -> a Volume per channel pair -> graph_out(C) -> master bus, 256-frame
blocks, 64 blocks per call, for C = 6 (5.1) and C = 8 (7.1). Prints one JSON line:

  * the device's name and power limit, read in this run;
  * ms per call (median, p10, p90 over --calls calls after warm-up; each call bracketed by CUDA events and synchronised on its own);
  * kernel launches per chunk (a call is one chunk here);
  * host time per block-sized call (one 256-frame block per call, replayed from the captured CUDA graph);
  * a 4-block prefix on a fresh context, bit-compared with the CPU oracle;
  * the bus launch's kernel time from a separate torch.profiler run, as GB/s over the V*C*T*4 bytes it reads and as a share of the
    H100 SXM data sheet's 3.35 TB/s; c2's bus launch (bench.py's c2 workload) is timed the same way in the same run for comparison.

Writes nothing to disk: the profiler's trace stays in memory."""
import argparse
import ctypes
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "oracle"))

HBM_PEAK_GBS = 3350.0  # NVIDIA H100 SXM data sheet (700 W part)
V, F, KB = 1024, 256, 64


def synth(shape, seed):
    rng = np.random.Generator(np.random.PCG64(seed))
    r = rng.integers(0, 1 << 24, size=shape, dtype=np.uint32)
    return (r.astype(np.float32) * np.float32(2.0 ** -24) * np.float32(2.0) - np.float32(1.0)).astype(np.float32)


def device_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    name, power, clk = (s.strip() for s in q.stdout.strip().splitlines()[0].split(","))
    return {"name": name, "power_limit": power, "max_sm_clock": clk}


def surround(fw, lib, C, V_, mcf=0):
    cx = fw.FirewheelGraphCtx(lib, fw.AudioGraphConfig(num_graph_inputs=C, num_graph_outputs=C, num_voices=V_, master_bus=True, max_call_frames=mcf))
    g = cx.graph
    rng = np.random.default_rng(C)
    for z in range(0, C, 2):
        w = min(2, C - z)
        vol = g.add_node(w, w, fw.VolumeNode(100.0))
        for c in range(w):
            g.connect(g.graph_in_node(), z + c, vol, c, False)
            g.connect(vol, c, g.graph_out_node(), z + c, False)
        g.set_percent_volume(vol, (20 + 100 * rng.random(V_)).astype(np.float32))
    proc = cx.activate(48000, C, C, F)
    st = cx.update()
    if st.graph_error is not None:
        raise RuntimeError(f"C={C}: {st.graph_error} {cx.last_error()}")
    return cx, proc


def bus_kernel_ms(proc, call, n):
    """mean device time per call of the bus launch (the BUS instantiation of chain_kernel), from torch.profiler's CUDA activities"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    call(); proc.sync()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(n):
            call()
        proc.sync()
    names, us = set(), 0.0
    for e in prof.events():
        if "chain_kernel" in e.name and "true" in e.name:
            names.add(e.name)
            us += e.device_time_total
    if not names:
        raise RuntimeError("the profiler saw no bus launch")
    return us / n / 1e3, sorted(names)


def run_surround(fw, lib, oracle, C, n_calls):
    T = F * KB
    cx, proc = surround(fw, lib, C, V)
    nbytes = V * C * T * 4
    h_in = lib.host_alloc_pinned(nbytes)
    h_out = lib.host_alloc_pinned(C * T * 4)
    x = np.ctypeslib.as_array(ctypes.cast(h_in, ctypes.POINTER(ctypes.c_float)), shape=(V, C, T))
    for v0 in range(0, V, 64):
        x[v0:v0 + 64] = synth((64, C, T), 0x5E0000 + C * 4096 + v0)
    d_in, d_out = lib.dev_malloc(0, nbytes), lib.dev_malloc(0, C * T * 4)
    if not d_in or not d_out:
        raise RuntimeError("device allocation failed")
    proc.h2d(d_in, h_in, nbytes); proc.sync()

    # 4-block prefix on this fresh context against the oracle
    Tp = 4 * F
    xp = np.ascontiguousarray(x[:, :, :Tp])
    yp = np.zeros((C, Tp), np.float32)
    rc, mp = proc.process_planar(xp, yp, C, C, Tp)
    assert rc == 0
    ocx, oproc = surround(fw, oracle, C, V)
    yo = np.zeros((C, Tp), np.float32)
    oproc.process_planar(xp, yo, C, C, Tp)
    oproc.free(); ocx.update(); ocx.free()
    parity = bool(np.array_equal(yp.view(np.uint32), yo.view(np.uint32)))

    def call():
        if proc.process_planar_device(d_in, d_out, C, C, T) != 0:
            raise RuntimeError(lib.last_device_error().decode())
    for _ in range(10):
        call()
    proc.sync()
    l0 = proc.kernel_launches()
    ms = []
    for _ in range(n_calls):
        proc.event_record(0); call(); proc.event_record(1); proc.sync()
        ms.append(proc.event_elapsed_ms(0, 1))
    launches = (proc.kernel_launches() - l0) / n_calls
    ms = np.array(ms)

    # block-sized calls: one 256-frame block per call, replayed from the captured CUDA graph
    n_block = 2000
    for _ in range(8):
        proc.process_planar_device(d_in, d_out, C, C, F)
    proc.sync()
    r0 = proc.graph_replays()
    t0 = time.perf_counter()
    for _ in range(n_block):
        proc.process_planar_device(d_in, d_out, C, C, F)
    proc.sync()
    host_us = (time.perf_counter() - t0) * 1e6 / n_block
    replays = proc.graph_replays() - r0

    k_ms, names = bus_kernel_ms(proc, call, 50)
    gbs = nbytes / (k_ms * 1e-3) / 1e9
    proc.free(); cx.update(); cx.free()
    lib.dev_free(0, d_in); lib.dev_free(0, d_out); lib.host_free_pinned(h_in); lib.host_free_pinned(h_out)
    return {"channels": C, "voices": V, "block_frames": F, "blocks_per_call": KB,
            "ms_per_call": float(np.median(ms)), "ms_per_call_p10": float(np.percentile(ms, 10)), "ms_per_call_p90": float(np.percentile(ms, 90)), "calls": n_calls,
            "launches_per_chunk": launches, "block_call_us_host": host_us, "block_call_graph_replays": replays,
            "parity_4_blocks_bit_exact": parity,
            "bus_kernel": {"names": names, "ms": k_ms, "bytes_read": nbytes, "GBps": gbs, "share_of_3350_GBps": gbs / HBM_PEAK_GBS}}


def run_c2(fw, lib):
    import bench
    w = bench.WORKLOADS["c2"]
    C, T = w["ch"], w["block"] * w["blocks"]
    cx, proc = bench.build_graph(fw, lib, "c2", V, w["block"], 0, 1000)
    nbytes = V * C * T * 4
    d_in, d_out = lib.dev_malloc(0, nbytes), lib.dev_malloc(0, C * T * 4)
    h_in = lib.host_alloc_pinned(nbytes)
    x = np.ctypeslib.as_array(ctypes.cast(h_in, ctypes.POINTER(ctypes.c_float)), shape=(V, C, T))
    for v0 in range(0, V, 64):
        x[v0:v0 + 64] = synth((64, C, T), 0xC20000 + v0)
    proc.h2d(d_in, h_in, nbytes); proc.sync()

    def call():
        if proc.process_planar_device(d_in, d_out, C, C, T) != 0:
            raise RuntimeError(lib.last_device_error().decode())
    for _ in range(10):
        call()
    k_ms, names = bus_kernel_ms(proc, call, 50)
    gbs = nbytes / (k_ms * 1e-3) / 1e9
    proc.free(); cx.update(); cx.free()
    lib.dev_free(0, d_in); lib.dev_free(0, d_out); lib.host_free_pinned(h_in)
    return {"voices": V, "channels": C, "frames_per_call": T, "bus_kernel": {"names": names, "ms": k_ms, "bytes_read": nbytes, "GBps": gbs, "share_of_3350_GBps": gbs / HBM_PEAK_GBS}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=200)
    ap.add_argument("--channels", default="6,8")
    args = ap.parse_args()
    import firewheel_b200 as fw
    import pyoracle
    lib, oracle = fw.load(), pyoracle.load()
    if lib.device_count() < 1:
        raise SystemExit("no CUDA device: " + lib.last_device_error().decode())
    res = {"device": device_info(), "surround": [run_surround(fw, lib, oracle, int(c), args.calls) for c in args.channels.split(",")], "c2": run_c2(fw, lib)}
    c2 = res["c2"]["bus_kernel"]["GBps"]
    for r in res["surround"]:
        r["bus_kernel"]["rate_vs_c2"] = r["bus_kernel"]["GBps"] / c2
    print(json.dumps(res))


if __name__ == "__main__":
    main()
