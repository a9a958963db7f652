"""Flat mixer on one GPU: the reference's everyday mixer as one flat graph (num_voices = 1) of V voices SamplerNode -> VolumeNode ->
PanNode, every other voice through a 2-stage biquad, under a balanced tree of 2-port SumNodes into graph_out; every voice loops its
own sample. For V in --voices (default 8, 32, 128), 256-frame blocks at 48 kHz, prints one JSON line per V:

  * the compiled schedule: nodes, pool buffers and smoothed parameters;
  * block-sized calls (one 256-frame block per call; steady, so replayed from the captured CUDA graph): median, p10 and p90 host time
    per call, and the median against the 5333 us a 256-frame block lasts at 48 kHz;
  * 64-block calls (one chunk each): median, p10 and p90 host time per call;
  * kernel launches per chunk, and the control kernel's time per call (processor_profile class 0, CUDA events) for both call sizes,
    next to the time of every other kernel class.

The device's name and power limit are read in the same run and printed first. Writes nothing to disk."""
import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

SR, F = 48000, 256
BUDGET_US = 1e6 * F / SR


def device_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    name, power, clk = (s.strip() for s in q.stdout.strip().splitlines()[0].split(","))
    return {"name": name, "power_limit": power, "max_sm_clock": clk}


def synth(shape, seed):
    rng = np.random.Generator(np.random.PCG64(seed))
    r = rng.integers(0, 1 << 24, size=shape, dtype=np.uint32)
    return (r.astype(np.float32) * np.float32(2.0 ** -24) * np.float32(2.0) - np.float32(1.0)).astype(np.float32)


def flat_mixer(fw, lib, V, kb):
    cx = fw.FirewheelGraphCtx(lib, fw.AudioGraphConfig(num_graph_inputs=0, num_graph_outputs=2, max_call_frames=kb * F))
    g = cx.graph
    rng = np.random.default_rng(V)
    leaves, smps, n_sm_of = [], [], {}  # n_sm_of: smoothed parameters per node id (sampler 1, volume 1, pan 2)
    for v in range(V):
        s, a, p = g.add_node(0, 2, fw.SamplerNode(100.0)), g.add_node(2, 2, fw.VolumeNode(float(20 + 80 * rng.random()))), g.add_node(2, 2, fw.PanNode(float(rng.uniform(-1, 1))))
        n_sm_of.update({int(s): 1, int(a): 1, int(p): 2})
        for c in range(2):
            g.connect(s, c, a, c, False)
            g.connect(a, c, p, c, False)
        last = p
        if v % 2:
            b = g.add_node(2, 2, fw.BiquadNode(2))
            g.set_biquad_coeffs(b, np.stack([fw.design_rbj(lib, 0, 400.0 + 30.0 * v, 0.7, 0.0, SR), fw.design_rbj(lib, 1, 80.0, 0.7, 0.0, SR)]).astype(np.float32))
            for c in range(2):
                g.connect(p, c, b, c, False)
            last = b
        leaves.append(last)
        smps.append(s)
    while len(leaves) > 1:
        nxt = []
        for i in range(0, len(leaves), 2):
            pair = leaves[i:i + 2]
            sn = g.add_node(2 * len(pair), 2, fw.SumNode())
            for k, leaf in enumerate(pair):
                for c in range(2):
                    g.connect(leaf, c, sn, 2 * k + c, False)
            nxt.append(sn)
        leaves = nxt
    for c in range(2):
        g.connect(leaves[0], c, g.graph_out_node(), c, False)
    sched, n_buf = g.compile_internal(F)
    proc = cx.activate(SR, 0, 2, F)
    st = cx.update()
    if st.graph_error is not None:
        raise RuntimeError(f"V={V}: {st.graph_error} {cx.last_error()}")
    res = [g.create_sample_resource(synth((2, 48000 + 1000 * i), i)) for i in range(4)]
    for v, s in enumerate(smps):
        g.sampler_set_sample(s, res[v % 4], True)
        g.sampler_set_loop_range(s, "full")
        g.sampler_play(s)
    return cx, proc, sched, n_buf, sum(n_sm_of.get(int(sn.id), 0) for sn in sched)


def timed_calls(proc, T, calls, warmup):
    out = np.zeros((2, T), np.float32)
    x = np.zeros((1, 0, T), np.float32)
    for _ in range(warmup):
        proc.process_planar(x, out, 0, 2, T)
    l0, r0 = proc.kernel_launches(), proc.graph_replays()
    us = []
    for _ in range(calls):
        t0 = time.perf_counter()
        rc, _ = proc.process_planar(x, out, 0, 2, T)  # host buffers: returns after the device has finished the call
        us.append(1e6 * (time.perf_counter() - t0))
        if rc != 0:
            raise RuntimeError(f"process_planar rc={rc}")
    launches = (proc.kernel_launches() - l0) / calls
    replays = proc.graph_replays() - r0
    proc.profile(True)  # class times in a separate pass: profiling runs the launches plainly, not from the captured graph
    ms = np.zeros(4)
    for _ in range(calls):
        proc.process_planar(x, out, 0, 2, T)
        ms += proc.profile_read()[0]  # read per call: the profiler holds a bounded number of launch scopes
    proc.profile(False)
    q = np.percentile(us, [10, 50, 90])
    return {"median_us": round(float(q[1]), 1), "p10_us": round(float(q[0]), 1), "p90_us": round(float(q[2]), 1),
            "launches_per_chunk": launches, "graph_replays": replays,
            "class_us_per_call": {name: round(1e3 * ms[i] / calls, 2) for i, name in enumerate(("control", "chain", "combine", "temporal"))}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--voices", default="8,32,128")
    ap.add_argument("--calls", type=int, default=400)
    ap.add_argument("--warmup", type=int, default=20)
    args = ap.parse_args()
    import firewheel_b200 as fw
    lib = fw.load()
    if lib.device_count() < 1:
        raise SystemExit("no CUDA device: " + lib.last_device_error().decode())
    print(json.dumps({"device": device_info()}), flush=True)
    for V in (int(s) for s in args.voices.split(",")):
        line = {"voices": V}
        for name, kb, calls in (("block_calls", 1, args.calls), ("calls_64_blocks", 64, max(20, args.calls // 8))):
            cx, proc, sched, n_buf, n_sm = flat_mixer(fw, lib, V, kb)
            line["schedule"] = {"nodes": len(sched), "buffers": n_buf, "smoothers": n_sm}
            r = timed_calls(proc, kb * F, calls, args.warmup)
            if kb == 1:
                r["median_vs_budget"] = round(r["median_us"] / BUDGET_US, 4)
            line[name] = r
            proc.free(); cx.update(); cx.free()
        line["budget_us"] = round(BUDGET_US, 1)
        print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
