"""Streams whose channel counts differ from the graph's ports, on one GPU: bench.py's c2 graph (1024 voices of graph_in(2) -> Volume ->
Pan -> graph_out(2) -> master bus, 256-frame blocks) on a 2-channel stream (matched) against the same graph on a 6- and an 8-channel
output stream (four and six +0.0 bus rows per call), and on a mono input stream (graph_in port 1 reads +0.0). The layouts run
alternately, round after round, for 64-block calls and block-sized calls (replayed from the captured CUDA graph). Prints one JSON line
with the device's name and power limit read in this run, and per layout and call size: ms per call (median, p10, p90 over every round's
calls; each call bracketed by CUDA events and synchronised on its own) and kernel launches per call. Writes nothing to disk."""
import argparse
import json
import subprocess
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

V, F = 1024, 256
LAYOUTS = {"matched_2in_2out": (2, 2), "six_out": (2, 6), "eight_out": (2, 8), "mono_in": (1, 2)}  # (n_in, n_out) of the stream


def device_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    name, power, clk = (s.strip() for s in q.stdout.strip().splitlines()[0].split(","))
    return {"name": name, "power_limit": power, "max_sm_clock": clk}


def c2(fw, lib, n_in, n_out):
    cx = fw.FirewheelGraphCtx(lib, fw.AudioGraphConfig(num_graph_inputs=2, num_graph_outputs=2, num_voices=V, master_bus=True))
    g = cx.graph
    vol, pn = g.add_node(2, 2, fw.VolumeNode(100.0)), g.add_node(2, 2, fw.PanNode(0.0))
    for c in range(2):
        g.connect(g.graph_in_node(), c, vol, c, False)
        g.connect(vol, c, pn, c, False)
        g.connect(pn, c, g.graph_out_node(), c, False)
    rng = np.random.default_rng(2)
    g.set_percent_volume(vol, (25 + 75 * rng.random(V)).astype(np.float32))
    g.set_pan(pn, rng.uniform(-1, 1, V).astype(np.float32))
    proc = cx.activate(48000, n_in, n_out, F)
    st = cx.update()
    if st.graph_error is not None:
        raise RuntimeError(f"{n_in}->{n_out}: {st.graph_error} {cx.last_error()}")
    return cx, proc


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--calls", type=int, default=40, help="timed calls per layout and round")
    args = ap.parse_args()
    import firewheel_b200 as fw
    lib = fw.load()
    if lib.device_count() < 1:
        raise RuntimeError("no CUDA device: " + lib.last_device_error().decode())
    result = {"device": device_info(), "voices": V, "block_frames": F}
    for blocks in (64, 1):
        T = blocks * F
        runs = {}
        for name, (n_in, n_out) in LAYOUTS.items():
            cx, proc = c2(fw, lib, n_in, n_out)
            d_in, d_out = lib.dev_malloc(0, max(1, V * n_in * T * 4)), lib.dev_malloc(0, n_out * T * 4)
            x = np.random.default_rng(7).uniform(-1, 1, (V, n_in, T)).astype(np.float32)
            proc.h2d(d_in, x.ctypes.data, x.nbytes)
            runs[name] = (cx, proc, d_in, d_out, n_in, n_out, [], [])
        def call(r):
            _, proc, d_in, d_out, n_in, n_out, _, _ = r
            if proc.process_planar_device(d_in, d_out, n_in, n_out, T) != 0:
                raise RuntimeError(lib.last_device_error().decode())
        for r in runs.values():  # warm-up: module loads, the CUDA-graph capture of the steady chunk
            for _ in range(10):
                call(r)
            r[1].sync()
        for _ in range(args.rounds):
            for r in runs.values():
                proc, ms, launches = r[1], r[6], r[7]
                for _ in range(args.calls):
                    l0 = proc.kernel_launches()
                    proc.event_record(0); call(r); proc.event_record(1); proc.sync()
                    ms.append(proc.event_elapsed_ms(0, 1)); launches.append(proc.kernel_launches() - l0)
        out = {}
        for name, (cx, proc, d_in, d_out, *_rest, ms, launches) in runs.items():
            ms = np.array(ms)
            out[name] = {"ms_median": float(np.median(ms)), "ms_p10": float(np.percentile(ms, 10)), "ms_p90": float(np.percentile(ms, 90)),
                         "launches_per_call": float(np.mean(launches)), "graph_replays": int(proc.graph_replays())}
            proc.free(); cx.update(); cx.free()
            lib.dev_free(0, d_in); lib.dev_free(0, d_out)
        result[f"{blocks}_block_calls"] = out
    print(json.dumps(result))


if __name__ == "__main__":
    main()
