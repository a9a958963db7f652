"""Graphs of any size on the device: flat mixers of many heterogeneous voices (hundreds of nodes, hundreds of pool buffers,
hundreds of smoothed parameters, many samplers and resamplers) and batched voice graphs with more than 16 smoothed parameters,
against the CPU oracle, bit for bit, outputs and silence masks.

The CPU test builds every graph the GPU tests use on the oracle and checks from the compiled schedule that, taken together, they are
large in every dimension the control plane sizes by the graph (nodes, buffers, ports, smoothers, samplers, resamplers, mask-dependent
nodes), so that the GPU tests keep covering what they claim to. It also checks that they cover every way the control kernel reads its
tables and keeps its silence flags (kernels.cu launch_control):
  * table image carried in the kernel parameters (up to 2 KB): the batched 9-PanNode graphs;
  * shared-memory copy of the device image: the 33-voice flat mixers;
  * device image read through L1 (image and flags over 48 KB): the 130-voice flat mixer;
  * fewer than 128 threads per CTA and shared memory beyond 48 KB (opt-in): the 1600-voice sampler graph (3200 pool buffers).

The chain kernel's warp fast path (all voices of a warp steady, every smoother REC_CONST) needs blocks of a multiple of 128 frames
(the 4-frame-per-lane tile) or 32 frames (1 frame per lane, unaligned calls): the tests that aim at it run 256-frame blocks."""
import numpy as np
import pytest

from conftest import synth
from firewheel_b200 import (AudioGraphConfig, BiquadNode, DelayNode, FirewheelGraphCtx, HardClipNode, MonoToStereoNode, PanNode,
                            ResamplerNode, SamplerNode, SumNode, SvfNode, VolumeNode, design_rbj, design_resampler, design_svf)
from helpers import SR, assert_bit_exact, f32, run_planar

F = 64                       # block frames, unless a test says otherwise
FB = 256                     # block frames of the tests that reach the chain kernel's warp fast path
MIXER_SIZES = (5, 17, 33, 130)
WALL_V = 1600                # voices of the sampler wall: 3200 pool buffers
BATCH_V = 37                 # voices of the batched contexts
N_PANS = 9                   # PanNodes of the batched voice graph: 18 smoothed parameters


# ---- graph builders (the same code drives the CUDA product and the CPU oracle) --------------------------------------------------
def flat_mixer(lib, V, delay=True, resampler=True, max_call_frames=4 * F, extra_voices=0, muted=True):
    """The reference's everyday mixer as one flat graph: per voice SamplerNode -> VolumeNode -> PanNode, every other voice through a
    2-stage biquad, some voices mono (SamplerNode(1) -> MonoToStereoNode), some through a HardClipNode, an SVF or a delay, some
    played by a ResamplerNode; a balanced tree of 2-port SumNodes into graph_out. Returns (cx, ids, kinds) where ids holds per-voice
    node ids and kinds maps every node id to its kind name. extra_voices: voices whose nodes are built but left out of the tree (see
    add_voice). muted = False: no voice starts muted (a muted voice keeps its VolumeNode's record REC_CLEAR)."""
    cx = FirewheelGraphCtx(lib, AudioGraphConfig(num_graph_inputs=0, num_graph_outputs=2, max_call_frames=max_call_frames))
    g = cx.graph
    kinds = {}
    rng = np.random.default_rng(V)
    table = design_resampler(lib, 64, 16) if resampler else None

    def add(ni, no, node, kind):
        nid = g.add_node(ni, no, node)
        kinds[int(nid)] = kind
        return nid

    def link(a, b, n=2):
        for c in range(n):
            g.connect(a, c, b, c, False)

    ids = {"src": [], "vol": [], "pan": [], "kind": [], "out": []}
    for v in range(V + extra_voices):
        if resampler and v % 16 == 5:
            src, kind = add(0, 2, ResamplerNode(table), "resampler"), "resampler"
            head = src
        elif v % 8 == 3:
            src, kind = add(0, 1, SamplerNode(100.0), "sampler"), "mono"
            head = add(1, 2, MonoToStereoNode(), "m2s")
            g.connect(src, 0, head, 0, False)
        else:
            src, kind = add(0, 2, SamplerNode(100.0), "sampler"), "sampler"
            head = src
        vol = add(2, 2, VolumeNode(100.0), "volume")
        pan = add(2, 2, PanNode(0.0), "pan")
        link(head, vol)
        link(vol, pan)
        last = pan
        if v % 2 == 1:
            bq = add(2, 2, BiquadNode(2), "biquad")
            g.set_biquad_coeffs(bq, np.stack([design_rbj(lib, 0, 500.0 + 40.0 * v, 0.7, 0.0, SR), design_rbj(lib, 1, 60.0, 0.7, 0.0, SR)]).astype(f32))
            link(last, bq)
            last = bq
        if v % 8 == 2:
            hc = add(2, 2, HardClipNode(-3.0), "hardclip")
            link(last, hc)
            last = hc
        if v % 8 == 6:
            svf = add(2, 2, SvfNode(1), "svf")
            g.set_svf_coeffs(svf, design_svf(lib, 0, 900.0 + 10.0 * v, 0.9, SR)[None, :])
            link(last, svf)
            last = svf
        if delay and v % 8 == 4:
            dl = add(2, 2, DelayNode(37 * (v % 5 + 1)), "delay")
            link(last, dl)
            last = dl
        pct = 0.0 if muted and v % 9 == 7 else float(20.0 + 80.0 * rng.random())   # a few voices start muted
        g.set_percent_volume(vol, pct)
        g.set_pan(pan, float(rng.uniform(-1.0, 1.0)))
        for k, x in (("src", src), ("vol", vol), ("pan", pan), ("kind", kind), ("out", last)):
            ids[k].append(x)
    ids["root"] = sum_tree(g, ids["out"][:V], kinds)
    link(ids["root"], g.graph_out_node())
    return cx, ids, kinds


def sum_tree(g, leaves, kinds, ports=2):
    """Balanced tree of `ports`-port stereo SumNodes over `leaves` (the last node of a level takes what is left, a 1-port SumNode copies)."""
    while len(leaves) > 1:
        nxt = []
        for i in range(0, len(leaves), ports):
            pair = leaves[i:i + ports]
            sn = g.add_node(2 * len(pair), 2, SumNode())
            kinds[int(sn)] = "sum"
            for k, leaf in enumerate(pair):
                for c in range(2):
                    g.connect(leaf, c, sn, 2 * k + c, False)
            nxt.append(sn)
        leaves = nxt
    return leaves[0]


def add_voice(g, ids, kinds, v):
    """Graph edit: voice v (built by flat_mixer(extra_voices=...)) joins the mix through a new 2-port SumNode after the tree root."""
    top = g.add_node(4, 2, SumNode())
    kinds[int(top)] = "sum"
    for c in range(2):
        g.disconnect(ids["root"], c, g.graph_out_node(), c)
        g.connect(ids["root"], c, top, c, False)
        g.connect(ids["out"][v], c, top, 2 + c, False)
        g.connect(top, c, g.graph_out_node(), c, False)
    ids["root"] = top


def make_resources(g):
    """Stereo, mono and short resources whose lengths end mid-block; -0.0 samples included."""
    def neg_zeros(a):
        a = a.copy()
        a[..., ::7] = -0.0
        return a
    return [g.create_sample_resource(neg_zeros(synth((2, 1000), 1))),
            g.create_sample_resource(synth((2, 5000), 2)),
            g.create_sample_resource(neg_zeros(synth((1, 777), 3))),
            g.create_sample_resource(synth((2, 90), 4))]


def start_voices(g, ids, res, voices=None):
    """Every voice plays: resource by voice, voices % 5 == 0 loop the whole sample, resampler voices at their own rate."""
    for v in (range(len(ids["src"])) if voices is None else voices):
        src, kind = ids["src"][v], ids["kind"][v]
        if kind == "resampler":
            g.resampler_set(src, res[v % 2], ratio=0.75 + 0.05 * (v % 7), playing=True, loop=(v % 3 == 0), voice=0)
            continue
        r = res[2] if kind == "mono" else res[v % 4 if v % 4 != 2 else 0]
        g.sampler_set_sample(src, r, True, voice=0)
        if v % 5 == 0:
            g.sampler_set_loop_range(src, "full", voice=0)
        g.sampler_play(src, voice=0)


def stamped(g, block, fn):
    g.set_event_block(block)
    fn()
    g.set_event_block(0)


def mixer_scenario(lib, V, delay=True, resampler=True):
    """Outputs and masks of a sequence of calls on the flat mixer: samples start, gain and pan ramps stamped mid-call, mutes, samples
    that end mid-call, calls longer than max_call_frames (chunked) and a partial last block."""
    cx, ids, _ = flat_mixer(lib, V, delay=delay, resampler=resampler)
    proc = cx.activate(SR, 0, 2, F)
    st = cx.update()
    assert st.kind == "Active" and st.graph_error is None, (st, cx.last_error())
    g = cx.graph
    res = make_resources(g)
    rng = np.random.default_rng(100 + V)

    def ramps():
        for v in range(0, V, 3):
            g.set_percent_volume(ids["vol"][v], float(10.0 + 90.0 * rng.random()))
            g.set_pan(ids["pan"][v], float(rng.uniform(-1.0, 1.0)))

    def mutes():
        for v in range(1, V, 4):
            g.set_percent_volume(ids["vol"][v], 0.0)

    def unmute():
        for v in range(1, V, 4):
            g.set_percent_volume(ids["vol"][v], 70.0)

    calls = [(lambda: start_voices(g, ids, res), 10 * F), (lambda: stamped(g, 3, ramps), 9 * F), (lambda: stamped(g, 5, mutes), 6 * F + 17),
             (None, 12 * F), (lambda: stamped(g, 2, unmute), 7 * F), (lambda: start_voices(g, ids, res), 11 * F), (None, 20 * F)]
    outs = []
    for act, T in calls:
        if act:
            act()
        outs.append(run_planar(proc, np.zeros((1, 0, T), f32), 2))
    proc.free(); cx.update(); cx.free()
    return outs


def batched_pans(lib, dag, block=F):
    """num_voices = 37 with a master bus; the voice graph holds 9 PanNodes (18 smoothed parameters). dag = False: a linear chain
    graph_in -> 9 x PanNode -> graph_out (fused-chain lowering); dag = True: the same 9 PanNodes in a row next to a dry VolumeNode,
    summed by a 2-port SumNode (generic lowering)."""
    cx = FirewheelGraphCtx(lib, AudioGraphConfig(num_graph_inputs=2, num_graph_outputs=2, num_voices=BATCH_V, master_bus=True,
                                                 max_call_frames=8 * block))
    g = cx.graph
    rng = np.random.default_rng(7)
    pans, prev = [], g.graph_in_node()
    for _ in range(N_PANS):
        p = g.add_node(2, 2, PanNode(0.0))
        for c in range(2):
            g.connect(prev, c, p, c, False)
        g.set_pan(p, rng.uniform(-1.0, 1.0, BATCH_V).astype(f32))
        pans.append(p)
        prev = p
    if dag:
        dry = g.add_node(2, 2, VolumeNode(60.0))
        mix = g.add_node(4, 2, SumNode())
        for c in range(2):
            g.connect(g.graph_in_node(), c, dry, c, False)
            g.connect(prev, c, mix, c, False)
            g.connect(dry, c, mix, 2 + c, False)
        prev = mix
    for c in range(2):
        g.connect(prev, c, g.graph_out_node(), c, False)
    return cx, pans


def sampler_wall(lib, V):
    """A flat graph of V stereo SamplerNodes under a tree of 32-port SumNodes: the compiler schedules every sampler first, so 2 V pool
    buffers are live at once."""
    cx = FirewheelGraphCtx(lib, AudioGraphConfig(num_graph_inputs=0, num_graph_outputs=2))
    g = cx.graph
    kinds, srcs = {}, []
    for _ in range(V):
        s = g.add_node(0, 2, SamplerNode(100.0))
        kinds[int(s)] = "sampler"
        srcs.append(s)
    root = sum_tree(g, list(srcs), kinds, ports=32)
    for c in range(2):
        g.connect(root, c, g.graph_out_node(), c, False)
    return cx, srcs, kinds


# ---- CPU: the graphs are as large as the tests claim ---------------------------------------------------------------------------
def schedule_counts(lib, cx, kinds):
    """What the device lowering derives from the product compiler's schedule (runtime.cu lower_control / lower_generic)."""
    sched, n_buf = cx.graph.compile_internal(F)
    n_sm, straddle, in_ports, out_ports, masks = 0, False, 0, 0, 0
    for i, sn in enumerate(sched):
        kind = kinds.get(int(sn.id), "endpoint")
        in_ports += len(sn.input_buffers)
        out_ports += len(sn.output_buffers)
        k = {"volume": 1, "sampler": 1, "pan": 2}.get(kind, 0)
        if kind == "pan" and n_sm % 16 == 15:
            straddle = True
        n_sm += k
        endpoint = i == 0 or i + 1 == len(sched)
        if not endpoint and sn.output_buffers and ((kind == "sum" and len(sn.input_buffers) != len(sn.output_buffers)) or kind in ("hardclip", "m2s")):
            masks += 1
    c = dict(nodes=len(sched), buffers=n_buf, in_ports=in_ports, out_ports=out_ports, ports=in_ports + out_ports, smoothers=n_sm,
             straddle=straddle, masks=masks, samplers=sum(kinds.get(int(s.id)) == "sampler" for s in sched),
             resamplers=sum(kinds.get(int(s.id)) == "resampler" for s in sched))
    c["control"] = control_modes(c)
    return c


def control_modes(c):
    """How the control kernel runs a plan of these counts, as launch_control decides it (kernels.cu) for an H100 (227 KB of opt-in
    shared memory). Element sizes are those of plan.hpp: CtlNode 24 B, a port 4 B, SmDesc 32 B, SamplerCtl 88 B, RsCtl 24 B."""
    r16 = lambda n: (n + 15) // 16 * 16
    image = (r16(24 * c["nodes"]) + r16(4 * c["in_ports"]) + r16(4 * c["out_ports"]) + r16(32 * c["smoothers"]) + r16(88 * c["samplers"])
             + r16(24 * c["resamplers"]))
    per_thread = 16 * (max(1, -(-c["buffers"] // 64)) - 1)   # flag words 1.., twice
    threads = 128
    if per_thread * 128 > 48 * 1024:
        threads = 64
        while per_thread * threads > 227 * 1024:
            threads //= 2
    flags = per_thread * threads
    staged = flags + image <= 48 * 1024
    modes = {"param" if staged and image <= 2048 else "shared" if staged else "global"}
    if threads < 128:
        modes.add("fewer_threads")
    if flags > 48 * 1024:
        modes.add("optin_smem")
    return modes


def test_graphs_exceed_every_former_device_limit(oracle):
    counts = []
    for V in MIXER_SIZES:
        cx, _, kinds = flat_mixer(oracle, V)
        counts.append(schedule_counts(oracle, cx, kinds))
        cx.free()
    cx, _, kinds = flat_mixer(oracle, 33, delay=False, resampler=False)
    counts.append(schedule_counts(oracle, cx, kinds))
    cx.free()
    for dag in (False, True):
        cx, pans = batched_pans(oracle, dag)
        kinds = {int(p): "pan" for p in pans}
        counts.append(schedule_counts(oracle, cx, kinds))
        assert counts[-1]["smoothers"] == 2 * N_PANS > 16
        cx.free()
    cx, _, kinds = sampler_wall(oracle, WALL_V)
    counts.append(schedule_counts(oracle, cx, kinds))
    cx.free()
    assert counts[-1]["buffers"] >= 2 * WALL_V, counts[-1]
    modes = [c["control"] for c in counts]
    assert all("param" in m for m in modes[-3:-1]), modes                            # the batched graphs
    assert "shared" in modes[MIXER_SIZES.index(33)] and "shared" in modes[len(MIXER_SIZES)], modes
    assert "global" in modes[MIXER_SIZES.index(130)], modes
    assert {"global", "fewer_threads", "optin_smem"} <= modes[-1], modes
    big = counts[MIXER_SIZES.index(130)]
    assert big["nodes"] > 64 and big["buffers"] > 256, big          # several silence-flag words per voice; buffer indices past 8 bits
    assert big["ports"] > 512, big
    assert big["smoothers"] > 32 and big["straddle"], big           # 16 per record word; a PanNode across a word boundary
    assert big["samplers"] > 4 and big["resamplers"] > 4, big
    assert big["masks"] > 32, big                                   # input-mask slots of the generic lowering
    small = counts[MIXER_SIZES.index(5)]
    assert small["smoothers"] > 16 and small["samplers"] > 4, small
    assert any(c["smoothers"] > 16 for c in counts[len(MIXER_SIZES):]), counts


# ---- GPU ---------------------------------------------------------------------------------------------------------------------------
def assert_same(og, oo):
    for i, ((yg, mg), (yo, mo)) in enumerate(zip(og, oo)):
        assert_bit_exact(yg, yo, f"call {i}")
        assert mg == mo, f"call {i}: silence mask {mg:#x} != {mo:#x}"


@pytest.mark.gpu
@pytest.mark.parametrize("V", MIXER_SIZES)
def test_flat_mixer_matches_oracle(gpu, oracle, V):
    og, oo = mixer_scenario(gpu, V), mixer_scenario(oracle, V)
    assert_same(og, oo)
    assert np.any(og[0][0] != 0)


@pytest.mark.gpu
def test_block_sized_calls_replay_and_recapture(gpu, oracle):
    """Without delay and resampler voices the plan is graphable: steady block-sized calls replay a captured CUDA graph; a sample
    resource created between calls changes the table the samplers read, so the chunk is captured anew. 256-frame blocks and no muted
    voice: the steady calls take the chain kernel's warp fast path, each PanNode's program staging two smoothers whose plan indices lie
    far beyond 16. The last two calls ramp one PanNode of the last voice (mode word 8 of 9): only the OR of every mode word in st_modes
    keeps the flat voice off the fast path."""
    V = 33
    outs, replays = [], []
    for lib in (gpu, oracle):
        cx, ids, _ = flat_mixer(lib, V, delay=False, resampler=False, max_call_frames=4 * FB, muted=False)
        proc = cx.activate(SR, 0, 2, FB)
        st = cx.update()
        assert st.kind == "Active" and st.graph_error is None, (st, cx.last_error())
        g = cx.graph
        res = make_resources(g)
        start_voices(g, ids, res)
        for v in range(V):  # loop every sampler so that the calls stay steady
            if ids["kind"][v] != "resampler":
                g.sampler_set_loop_range(ids["src"][v], "full", voice=0)
        seq, rp = [], []
        for i in range(16):
            if i == 8:
                g.create_sample_resource(synth((2, 300), 9))
            seq.append(run_planar(proc, np.zeros((1, 0, FB), f32), 2))
            rp.append(proc.graph_replays() if lib is gpu else 0)
        g.set_pan(ids["pan"][V - 1], -0.9, voice=0)
        seq += [run_planar(proc, np.zeros((1, 0, FB), f32), 2) for _ in range(2)]
        outs.append(seq); replays.append(rp)
        proc.free(); cx.update(); cx.free()
    assert_same(*outs)
    rp = replays[0]
    assert rp[7] > 0 and rp[7] > rp[3], rp                 # captured, then replayed
    assert rp[8] == rp[7] and rp[9] == rp[8] + 1, rp       # new table: first sight runs plainly, the second is captured and launched
    assert rp[15] == rp[9] + 6, rp


@pytest.mark.gpu
def test_graph_edit_adds_a_voice(gpu, oracle):
    """A voice joins the mix between calls: the schedule is swapped (first block of the new schedule reads a zeroed pool, Q11)."""
    V = 33
    outs = []
    for lib in (gpu, oracle):
        cx, ids, kinds = flat_mixer(lib, V, extra_voices=1)
        proc = cx.activate(SR, 0, 2, F)
        st = cx.update()
        assert st.kind == "Active" and st.graph_error is None, (st, cx.last_error())
        g = cx.graph
        res = make_resources(g)
        start_voices(g, ids, res)
        seq = [run_planar(proc, np.zeros((1, 0, T), f32), 2) for T in (5 * F, 3 * F)]
        add_voice(g, ids, kinds, V)
        st = cx.update()
        assert st.graph_error is None, (st, cx.last_error())
        start_voices(g, ids, res, voices=[V])
        seq += [run_planar(proc, np.zeros((1, 0, T), f32), 2) for T in (6 * F, 9 * F)]
        outs.append(seq)
        proc.free(); cx.update(); cx.free()
    assert_same(*outs)


@pytest.mark.gpu
def test_process_interleaved(gpu, oracle):
    V = 17
    outs = []
    for lib in (gpu, oracle):
        cx, ids, _ = flat_mixer(lib, V)
        proc = cx.activate(SR, 0, 2, F)
        st = cx.update()
        assert st.kind == "Active" and st.graph_error is None, (st, cx.last_error())
        g = cx.graph
        start_voices(g, ids, make_resources(g))
        seq = []
        for T in (7 * F, 3 * F + 5, 10 * F):
            out = np.full((T, 2), np.nan, f32)
            rc = proc.process_interleaved(np.zeros((0,), f32), out, 0, 2, T)
            assert rc == 0, (rc, lib.last_device_error())
            seq.append(out)
        outs.append(seq)
        proc.free(); cx.update(); cx.free()
    for i, (a, b) in enumerate(zip(*outs)):
        assert_bit_exact(a, b, f"call {i}")


@pytest.mark.gpu
@pytest.mark.parametrize("dag", [False, True], ids=["chain", "dag"])
def test_batched_voice_graph_over_16_smoothers(gpu, oracle, dag):
    """37 voices, master bus, 256-frame blocks, a voice graph with 18 smoothed parameters: modes span two record words and the chain
    programs are split so that none reads more than 16 smoothers (PanNodes 0-7, then PanNode 8 with plan smoothers 16 and 17 at
    program-local 0 and 1). Call 0: every voice steady from block 0 (pans set before activation start unsmoothed), so every warp takes
    the chain kernel's fast path in both programs. Call 1: only PanNode 8 of voices 5 and 30 ramps (mode word 1 only), still ramping at the
    call's end, while the other warps stay on the fast path. Calls 2-3: ramps on half the PanNodes of every voice, then a long chunked
    call in which they settle and later chunks are steady again. Call 4: an unaligned call (1 frame per lane, the other instantiation).
    Call 5: -0.0 inputs."""
    x = synth((BATCH_V, 2, 48 * FB), 11)
    outs = []
    for lib in (gpu, oracle):
        cx, pans = batched_pans(lib, dag, block=FB)
        proc = cx.activate(SR, 2, 2, FB)
        st = cx.update()
        assert st.kind == "Active" and st.graph_error is None, (st, cx.last_error())
        g = cx.graph
        rng = np.random.default_rng(3)
        seq = [run_planar(proc, x[:, :, :8 * FB].copy(), 2, True)]
        stamped(g, 3, lambda: [g.set_pan(pans[8], -0.5, voice=v) for v in (5, 30)])
        seq.append(run_planar(proc, x[:, :, 8 * FB:16 * FB].copy(), 2, True))
        stamped(g, 2, lambda: [g.set_pan(p, rng.uniform(-1.0, 1.0, BATCH_V).astype(f32)) for p in pans[::2]])
        seq.append(run_planar(proc, x[:, :, :12 * FB].copy(), 2, True))
        seq.append(run_planar(proc, x[:, :, :48 * FB].copy(), 2, True))
        seq.append(run_planar(proc, x[:, :, 3:3 + 16 * FB - 3].copy(), 2, True))
        seq.append(run_planar(proc, -np.zeros((BATCH_V, 2, 4 * FB), f32), 2, True))
        outs.append(seq)
        proc.free(); cx.update(); cx.free()
    assert_same(*outs)


@pytest.mark.gpu
def test_sampler_wall_of_3200_buffers(gpu, oracle):
    """1600 sampler voices in one flat graph: 3200 live pool buffers, 50 silence-flag words per voice. The control kernel runs with fewer
    than 128 threads per CTA and more than 48 KB of shared memory, and reads its 250 KB table image from device memory. Samples end
    mid-call (flags change), then the calls settle."""
    outs = []
    for lib in (gpu, oracle):
        cx, srcs, _ = sampler_wall(lib, WALL_V)
        proc = cx.activate(SR, 0, 2, F)
        st = cx.update()
        assert st.kind == "Active" and st.graph_error is None, (st, cx.last_error())
        g = cx.graph
        res = make_resources(g)
        for v, s in enumerate(srcs):
            g.sampler_set_sample(s, res[v % 4], True, voice=0)
            g.sampler_play(s, voice=0)
        outs.append([run_planar(proc, np.zeros((1, 0, T), f32), 2) for T in (10 * F, 8 * F + 9, 20 * F, 4 * F)])
        proc.free(); cx.update(); cx.free()
    assert_same(*outs)
    assert np.any(outs[0][0][0] != 0)
