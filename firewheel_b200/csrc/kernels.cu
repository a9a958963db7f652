// kernels.cu — sm_90a kernels for the per-block audio-graph DSP path.
//
//   control_kernel       K-ctl        per-voice control pass: silence flags, smoothers, sampler transport -> records
//   chain_kernel         K-chain      fused pointwise voice chain (+ master-bus tree), the HBM-bound headline kernel
//   sum_kernel           K-sum        multi-port SumNode on pool buffers (generic lowering)
//   silence_fix_kernel   K-fix        +0.0 where the reference's non-fused bodies clear flagged channels (generic lowering)
//   sampler_kernel       K-sampler    SamplerNode: resource fetch + conversion + gain
//   resampler_*_kernel   K-resampler  polyphase windowed-sinc sample player (+ seek / advance helpers)
//   combine_kernel       K-combine    radix-16 levels of the bus tree over partial buses
//   (de)interleave, fill, zero_rows, bus_mask    stream boundary and small helpers
// temporal.cu holds the biquad / SVF / delay kernels (biquad_delay_lanes; biquad_delay_generic / svf_generic, the scalar path), reverb.cu the wgmma FIR GEMM, exchange.cu the stream hand-over of the master-bus exchange.
//
// Bit-exactness rules (SURVEY.md §7 H2): this TU is compiled with --fmad=false, -ftz=false,
// -prec-div=true; recurrences additionally spell out __fmul_rn/__fadd_rn. Sum order equals the
// graph's association order: no atomics, no order-agnostic shuffles on sample data.
#include <cuda_runtime.h>

#include <cstdint>
#include <cstdlib>

#include "../../include/fw_b200.h"
#include "device.cuh"
#include "kernels.cuh"
#include "plan.hpp"

namespace fw {

// =============================================================================================
// K-ctl: per-voice control pass. One thread per voice walks the compiled schedule block by block
// and restates the reference's control logic, emitting records for the data kernels.
//   executor flags      schedule.rs:305-341
//   ParamSmoother       smoother.rs:115-194 (Q1-Q3, Q10 stall)
//   VolumeProcessor     volume.rs:92-110      SumNodeProcessor masks  sum.rs:52-65
//   MonoToStereo        mono_to_stereo.rs:41  StereoToMono stereo_to_mono.rs:41-47
//   HardClip masks      hard_clip.rs:60-93
// Only state transitions and gain curves are computed here; no sample data is touched.
// =============================================================================================
struct SmLocal { float input, last; uint32_t status; };

__device__ __forceinline__ uint64_t all_silent_mask(uint32_t n) { return n >= 64 ? ~0ull : ((1ull << n) - 1ull); }
__device__ __forceinline__ bool all_channels_silent(uint64_t m, uint32_t n) { uint64_t a = all_silent_mask(n); return (m & a) == a; }

__device__ __forceinline__ void sm_reset(SmLocal& s, float val, bool& changed) {  // smoother.rs:115-129
    if (s.status != SM_INACTIVE) { s.status = SM_INACTIVE; s.input = val; s.last = val; changed = true; }
    else if (s.input != val) { s.input = val; s.last = val; changed = true; }
}

// set_and_process (smoother.rs:133-140,159-194). Returns the record mode; *first = values[0].
__device__ __forceinline__ uint32_t sm_set_and_process(SmLocal& s, float val, uint32_t frames, float a, float b, float eps,
                                                       float* curve, float* const_val, bool* smoothing, bool& changed) {
    if (!(s.input == val)) { s.input = val; s.status = SM_ACTIVE; changed = true; }
    if (s.status != SM_ACTIVE || frames == 0) {  // Q1: the constant buffer (== input for any non-Active state)
        *const_val = s.input; *smoothing = s.status != SM_INACTIVE;
        return REC_CONST;
    }
    const float t = __fmul_rn(s.input, a);
    const float y0 = __fadd_rn(t, __fmul_rn(s.last, b));
    *smoothing = true;
    if (fabsf(__fsub_rn(s.input, y0)) < eps) {  // Q3: settle test on output[0]; reset() overwrites the whole curve
        s.last = s.input; s.status = SM_DEACTIVATING;  // Q2: stays Deactivating forever
        changed = true;
        *const_val = s.input;
        return REC_CONST;
    }
    if (y0 == s.last) {  // Q10: f32 fixed point outside epsilon — the curve is constant and no state changes
        *const_val = y0;
        return REC_CONST;
    }
    float y = y0;
    curve[0] = y0;
    for (uint32_t i = 1; i < frames; ++i) { y = __fadd_rn(t, __fmul_rn(y, b)); curve[i] = y; }
    s.last = y;
    changed = true;
    *const_val = y0;
    return REC_CURVE;
}

__device__ __forceinline__ SmLocal sm_load(const SmDesc& d, uint32_t v) { SmLocal s; s.input = d.input[v]; s.last = d.last[v]; s.status = d.status[v]; return s; }
__device__ __forceinline__ void sm_store(const SmDesc& d, uint32_t v, const SmLocal& s) { d.input[v] = s.input; d.last[v] = s.last; d.status[v] = s.status; }

// ---- SamplerNode control (sampler.rs:331-516) ----
struct SmpLocal { uint32_t playing, flags, res; uint64_t playhead, ls, le; };
__device__ __forceinline__ SmpLocal smp_load(const SamplerCtl& sc, uint32_t v) {
    SmpLocal q;
    q.playing = sc.playing[v]; q.playhead = sc.playhead[v]; q.flags = sc.loop_flags[v]; q.ls = sc.loop_start[v]; q.le = sc.loop_end[v]; q.res = sc.res[v];
    return q;
}
__device__ __forceinline__ void smp_store(const SamplerCtl& sc, uint32_t v, const SmpLocal& q) {
    sc.playing[v] = q.playing; sc.playhead[v] = q.playhead; sc.loop_flags[v] = q.flags; sc.loop_start[v] = q.ls; sc.loop_end[v] = q.le; sc.res[v] = q.res;
}

// the message drain of sampler.rs:331-414, for one voice
__device__ __forceinline__ void smp_apply_messages(SmpLocal& q, const SamplerCtl& sc, uint32_t v, const ResDesc* res_tab, uint32_t n_res) {
    for (uint32_t i = sc.msg_off[v]; i < sc.msg_off[v + 1]; ++i) {
        const SamplerMsgDev m = sc.msgs[i];
        const uint64_t loop_start_or_zero = (q.flags & 1u) ? q.ls : 0ull;
        switch (m.kind) {
            case SMSG_SET_SAMPLE:  // :333-364
                q.res = m.a;
                if ((q.flags & 3u) == 3u && q.res != 0 && q.res <= n_res) { q.ls = 0; q.le = res_tab[q.res - 1].frames; }  // update_sample :269-281
                if (m.x) { q.playhead = loop_start_or_zero; q.playing = 0; }
                break;
            case SMSG_PLAY: q.playing = 1; break;    // :365-371
            case SMSG_PAUSE: q.playing = 0; break;   // :372-378
            case SMSG_STOP: q.playhead = loop_start_or_zero; q.playing = 0; break;  // :379-391
            case SMSG_SET_PLAYHEAD: q.playhead = m.x; break;  // :392-399
            default:  // SMSG_SET_LOOP :400-412
                if (m.a == 0) { q.flags = 0; break; }
                if (m.a == 1) { q.flags = 3u; q.ls = 0; q.le = (q.res != 0 && q.res <= n_res) ? res_tab[q.res - 1].frames : 0ull; }
                else { q.flags = 1u; q.ls = m.x; q.le = m.y; }
                if (q.playhead >= q.ls && q.playhead < q.le) q.playhead = q.ls;
                break;
        }
    }
}

// the playing branch of sampler.rs:445-516: advances the playhead by one block, says what the block plays.
// Returns false when the block is cleared instead (non-looping sample already at its end).
__device__ __forceinline__ bool smp_step(SmpLocal& q, uint64_t len, uint32_t frames, SmpRec* r, bool& changed) {
    if (q.flags & 1u) {  // :445-484
        if (q.playhead >= q.le) q.playhead = q.ls;
        const uint64_t left = q.le - q.playhead;
        const uint32_t first = left < (uint64_t)frames ? (uint32_t)left : frames;
        r->p0 = q.playhead; r->first = first;
        if (first < frames) { q.playhead = q.ls + (frames - first); r->mode = SMP_PLAY_WRAP; }
        else { q.playhead += frames; r->mode = SMP_PLAY; }
        return true;
    }
    if (q.playhead >= len) { q.playing = 0; changed = true; r->p0 = 0; r->first = 0; r->mode = SMP_CLEAR; return false; }  // :486-497
    const uint64_t left = len - q.playhead;
    const uint32_t copy = left < (uint64_t)frames ? (uint32_t)left : frames;
    r->p0 = q.playhead; r->first = copy;
    if (copy < frames) { q.playing = 0; q.playhead = 0; changed = true; r->mode = SMP_PLAY_ZERO_TAIL; }  // :503-513
    else { q.playhead += frames; r->mode = SMP_PLAY; }
    return true;
}

// The tables are device arrays of any size; per-voice state stays where it lives (smoothers, sampler transport: read and written in
// place). The silence flags of the voice are n_flag_words words: word 0 (pool buffers 0-63) in a register, words 1.. — a graph of
// more than 64 buffers — in shared memory, s_dyn[0][w - 1][thread] during the block and s_dyn[1][w - 1][thread] their value at its
// start. When it fits (stage_tables), the table image follows them in shared memory: one parallel copy per CTA, from the kernel
// parameters when the image travels there, instead of a chain of dependent global loads per node.
__global__ void __launch_bounds__(128) control_kernel(const __grid_constant__ ControlArgs a) {
    pdl_launch_dependents();  // the data kernel may start loading samples now; it waits for us before reading records
    extern __shared__ __align__(16) uint64_t s_dyn[];
    const CtlTables& tb = a.tables;
    const uint32_t W = tb.n_flag_words, B = blockDim.x;
    const char* tab = static_cast<const char*>(tb.image);
    if (a.stage_tables) {  // the tables do not change while the plan lives: copied before waiting for the previous kernel
        uint32_t* d = reinterpret_cast<uint32_t*>(s_dyn + 2 * (size_t)(W - 1) * B);
        const uint32_t* s = static_cast<const uint32_t*>(a.image_in_param ? static_cast<const void*>(a.image) : tb.image);
        for (uint32_t i = threadIdx.x; i < tb.image_bytes / 4; i += B) d[i] = s[i];
        tab = reinterpret_cast<const char*>(d);
        __syncthreads();
    }
    pdl_wait();               // the previous call's data kernels still read the record buffers we are about to rewrite
    const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t V = a.num_voices;
    if (v >= V) return;
    const CtlNode* const nodes = reinterpret_cast<const CtlNode*>(tab + tb.o_nodes);
    const uint32_t* const in_port = reinterpret_cast<const uint32_t*>(tab + tb.o_in_port);
    const uint32_t* const out_port = reinterpret_cast<const uint32_t*>(tab + tb.o_out_port);
    const SmDesc* const smd = reinterpret_cast<const SmDesc*>(tab + tb.o_sm);
    const SamplerCtl* const smp = reinterpret_cast<const SamplerCtl*>(tab + tb.o_smp);
    const RsCtl* const rsc = reinterpret_cast<const RsCtl*>(tab + tb.o_rs);
    const uint32_t F = a.block_frames, NSMP = tb.n_samplers, MW = a.rec.n_mode_words;
    const uint32_t n_blocks = (a.frames + F - 1) / F;
    uint64_t* const fl = s_dyn + threadIdx.x;            // word w >= 1: fl[(w - 1) * B]
    uint64_t* const fl0 = fl + (size_t)(W - 1) * B;       // its value at the start of the block

    if (a.smp_msgs) {
        for (uint32_t s = 0; s < NSMP; ++s) {
            const SamplerCtl& sc = smp[s];
            SmpLocal q = smp_load(sc, v);
            smp_apply_messages(q, sc, v, a.res_tab, a.n_res);
            smp_store(sc, v, q);
        }
    }
    uint64_t f0 = a.flags[v];
    for (uint32_t w = 1; w < W; ++w) fl[(w - 1) * B] = a.flags[(size_t)w * V + v];
    uint64_t gout_mask = 0;
    uint32_t steady = 0xffffffffu, k = 0, last_modes = 0, slot = 0;
    bool steady_mode = false;

    for (; k < n_blocks; ++k) {
        const uint32_t frames = min(F, a.frames - k * F);
        if (steady_mode) {
            // Nothing but sampler playheads moves. The block replays the steady record unless a non-looping sample
            // reaches its end in it (sampler.rs:486-513), which starts a new transient.
            bool evt = false;
            for (uint32_t s = 0; s < NSMP; ++s) {
                const SamplerCtl& sc = smp[s];
                if (!sc.last_play[v]) continue;
                const uint32_t res = sc.res[v];
                if (!(sc.loop_flags[v] & 1u) && sc.playhead[v] + frames > a.res_tab[res - 1].frames) evt = true;
            }
            if (!evt) {
                for (uint32_t s = 0; s < NSMP; ++s) {
                    const SamplerCtl& sc = smp[s];
                    SmpRec r; r.p0 = 0; r.first = 0; r.mode = SMP_CLEAR;
                    if (sc.last_play[v]) {
                        SmpLocal q = smp_load(sc, v);
                        bool dummy = false;
                        smp_step(q, a.res_tab[q.res - 1].frames, frames, &r, dummy);
                        sc.playhead[v] = q.playhead;  // the only field a replayed block moves
                    }
                    Records::at_kv(sc.rec, k, v, V) = r;
                }
                Records::at_kv(a.rec.slot_of, k, v, V) = (uint16_t)slot;
                continue;
            }
            steady_mode = false; steady = 0xffffffffu; ++slot;
        }
        if (slot >= a.rec.kt_max) { *a.rec.error = a.err_value; break; }
        bool changed = false;  // smoother / sampler transport state moved during this block
        const uint64_t f0_start = f0;  // the block is a pure function of (flags, that state): equal at both ends => it replays
        for (uint32_t w = 1; w < W; ++w) fl0[(w - 1) * B] = fl[(w - 1) * B];
        // Mode words of this record: smoothers are numbered in schedule order, so the walk meets them word by word and each word
        // is stored once, when the walk has moved past it.
        uint32_t mw = 0, mword = 0, mor = 0;
        auto put_mode = [&](int32_t s, uint32_t m) {
            const uint32_t w = (uint32_t)s / kModesPerWord;
            for (; mw < w; ++mw) { a.rec.mode_word(slot, mw, v, V) = mword; mor |= mword; mword = 0; }
            mword |= m << (2 * ((uint32_t)s % kModesPerWord));
        };
        auto put_val = [&](int32_t s, float cv) {
            a.rec.val(slot, s, v, V) = cv;
            a.rec.st_val(s, v, V) = cv;  // the last value written is the steady record's
        };
        auto curve_of = [&](int32_t s) { return a.rec.curve(slot, s, v, V, F); };
        for (uint32_t n = 0; n < tb.n_nodes; ++n) {
            const CtlNode nd = nodes[n];
            uint64_t in_mask = 0;
            for (uint32_t i = 0; i < nd.n_in; ++i) {  // schedule.rs:305-320
                const uint32_t pb = in_port[nd.in_off + i], b = pb & ~kPortClear;
                const uint64_t bit = 1ull << (b & 63u);
                bool set;
                if (b < 64u) { if (pb & kPortClear) f0 |= bit; set = (f0 & bit) != 0; }
                else { uint64_t& word = fl[((b >> 6) - 1) * B]; if (pb & kPortClear) word |= bit; set = (word & bit) != 0; }
                if (set) in_mask |= 1ull << i;
            }
            if (nd.mask_slot) {
                a.rec.in_mask(slot, nd.mask_slot - 1, v, V) = in_mask;
                a.rec.st_in_mask(nd.mask_slot - 1, v, V) = in_mask;  // the last mask written is the steady record's
            }
            uint64_t out_mask = 0;  // processor.rs:233 NONE_SILENT
            switch (nd.kind) {
                case FW_NODE_VOLUME: {
                    const SmDesc d = smd[nd.sm0];
                    SmLocal s = sm_load(d, v);
                    bool ch = false;
                    const float g = d.target[v];  // volume.rs:92
                    if (all_channels_silent(in_mask, nd.n_in)) {  // volume.rs:94-100
                        sm_reset(s, g, ch);
                        put_mode(nd.sm0, REC_CLEAR);
                        out_mask = all_silent_mask(nd.n_out);
                    } else {
                        float cv; bool smoothing;
                        uint32_t m = sm_set_and_process(s, g, frames, a.a, a.b, a.eps, curve_of(nd.sm0), &cv, &smoothing, ch);
                        if (!smoothing && cv < 0.00001f) {  // volume.rs:104-108
                            m = REC_CLEAR; out_mask = all_silent_mask(nd.n_out);
                        } else {
                            out_mask = in_mask;  // volume.rs:110
                        }
                        put_mode(nd.sm0, m);
                        put_val(nd.sm0, cv);
                    }
                    if (ch) { sm_store(d, v, s); changed = true; }
                    break;
                }
                case FW_NODE_PAN: {
                    const SmDesc dl = smd[nd.sm0], dr = smd[nd.sm1];
                    SmLocal sl = sm_load(dl, v), sr = sm_load(dr, v);
                    bool chl = false, chr = false;
                    const float gl = dl.target[v], gr = dr.target[v];
                    if (all_channels_silent(in_mask, nd.n_in)) {
                        sm_reset(sl, gl, chl); sm_reset(sr, gr, chr);
                        put_mode(nd.sm0, REC_CLEAR); put_mode(nd.sm1, REC_CLEAR);
                        out_mask = all_silent_mask(nd.n_out);
                    } else {
                        float cv; bool smoothing;
                        uint32_t m = sm_set_and_process(sl, gl, frames, a.a, a.b, a.eps, curve_of(nd.sm0), &cv, &smoothing, chl);
                        put_mode(nd.sm0, m);
                        put_val(nd.sm0, cv);
                        m = sm_set_and_process(sr, gr, frames, a.a, a.b, a.eps, curve_of(nd.sm1), &cv, &smoothing, chr);
                        put_mode(nd.sm1, m);
                        put_val(nd.sm1, cv);
                        out_mask = in_mask;
                    }
                    if (chl) { sm_store(dl, v, sl); changed = true; }
                    if (chr) { sm_store(dr, v, sr); changed = true; }
                    break;
                }
                case FW_NODE_SAMPLER: {  // sampler.rs:416-559
                    const SamplerCtl& sc = smp[nd.sm1];
                    SmpLocal q = smp_load(sc, v);
                    SmpRec r; r.p0 = 0; r.first = 0; r.mode = SMP_CLEAR;
                    bool play = false; uint32_t sch = 0;
                    if (q.res != 0 && q.res <= a.n_res && q.playing) {
                        const ResDesc rd = a.res_tab[q.res - 1];
                        sch = rd.channels;
                        const SmDesc d = smd[nd.sm0];
                        SmLocal s = sm_load(d, v);
                        bool ch = false;
                        float cv; bool smoothing;
                        const uint32_t m = sm_set_and_process(s, d.target[v], frames, a.a, a.b, a.eps, curve_of(nd.sm0), &cv, &smoothing, ch);  // :432-433
                        if (ch) { sm_store(d, v, s); changed = true; }
                        put_mode(nd.sm0, m);
                        put_val(nd.sm0, cv);
                        if (smoothing || !(cv < 0.00001f)) {  // :437-443 muted => clear, playhead stays
                            play = smp_step(q, rd.frames, frames, &r, changed);
                            smp_store(sc, v, q);
                        }
                    }
                    if (!play) out_mask = all_silent_mask(nd.n_out);
                    else if (nd.n_out > sch && !(nd.n_out == 2 && sch == 1))  // :545-559: channels past the sample's are zeroed and flagged
                        out_mask = all_silent_mask(nd.n_out) & ~all_silent_mask(sch);
                    sc.last_play[v] = play ? 1u : 0u;
                    Records::at_kv(sc.rec, k, v, V) = r;
                    break;
                }
                case FW_NODE_RESAMPLER: {  // spec ours: cleared + flagged when not playing / no resource; surplus channels as the sampler's
                    const RsCtl rc = rsc[nd.sm1];
                    const uint32_t r = rc.res[v];
                    if (!(rc.flags[v] & 1u) || r == 0 || r > a.n_res) out_mask = all_silent_mask(nd.n_out);
                    else { const uint32_t sch = a.res_tab[r - 1].channels; if (nd.n_out > sch && !(nd.n_out == 2 && sch == 1)) out_mask = all_silent_mask(nd.n_out) & ~all_silent_mask(sch); }
                    break;
                }
                case FW_NODE_SUM:  // sum.rs:52-65; the unrolled / generic sums never write the mask (Q7)
                    if (all_channels_silent(in_mask, nd.n_in)) out_mask = all_silent_mask(nd.n_out);
                    else if (nd.n_in == nd.n_out) out_mask = in_mask;
                    break;
                case FW_NODE_MONO_TO_STEREO:  // mono_to_stereo.rs:41-44
                    if (in_mask & 1ull) out_mask = all_silent_mask(nd.n_out);
                    break;
                case FW_NODE_STEREO_TO_MONO:  // stereo_to_mono.rs:41-47
                    if (all_channels_silent(in_mask, 2) || nd.n_in < 2 || nd.n_out == 0) out_mask = all_silent_mask(nd.n_out);
                    break;
                case FW_NODE_HARD_CLIP:  // hard_clip.rs:60-80 leaves the mask untouched on the stereo fast path
                    if (!(nd.n_in == 2 && nd.n_out == 2 && (in_mask & 3ull) == 0)) out_mask = in_mask;
                    break;
                case FW_NODE_CUSTOM:  // the plugin's declared out_silence_rule (include/fw_b200.h)
                    if (nd.sm0 == FW_OUT_SILENCE_PASSTHROUGH) out_mask = in_mask & all_silent_mask(nd.n_out);
                    else if (nd.sm0 == FW_OUT_SILENCE_ALL_IF_ALL_INPUTS && nd.n_in > 0 && all_channels_silent(in_mask, nd.n_in)) out_mask = all_silent_mask(nd.n_out);
                    break;
                default: break;  // dummy / graph_in / graph_out / biquad / delay / reverb: NONE_SILENT
            }
            if (n + 1 == tb.n_nodes) gout_mask = in_mask;  // graph_out is scheduled last (compiler.rs:291)
            for (uint32_t i = 0; i < nd.n_out; ++i) {  // schedule.rs:338-341
                const uint32_t b = out_port[nd.out_off + i];
                const uint64_t bit = 1ull << (b & 63u);
                const bool set = (out_mask >> i) & 1ull;
                if (b < 64u) f0 = set ? (f0 | bit) : (f0 & ~bit);
                else { uint64_t& word = fl[((b >> 6) - 1) * B]; word = set ? (word | bit) : (word & ~bit); }
            }
        }
        for (; mw < MW; ++mw) { a.rec.mode_word(slot, mw, v, V) = mword; mor |= mword; mword = 0; }
        last_modes = mor;
        if (a.rec.slot_of) Records::at_kv(a.rec.slot_of, k, v, V) = (uint16_t)slot;
        bool same = f0 == f0_start;
        for (uint32_t w = 1; w < W; ++w) same = same && fl0[(w - 1) * B] == fl[(w - 1) * B];
        if (!changed && same) {  // nothing moved: later blocks replay this record
            steady = k;
            if (NSMP == 0) break;
            steady_mode = true;
        } else {
            ++slot;
        }
    }
    if (steady == 0xffffffffu) steady = (k == 0 ? 0 : min(k, n_blocks) - 1);
    a.rec.steady_k[v] = steady;
    a.rec.st_modes[v] = last_modes;  // the record of block `steady`: any smoother not REC_CONST
    a.rec.gout_mask[v] = gout_mask;
    a.flags[v] = f0;
    for (uint32_t w = 1; w < W; ++w) a.flags[(size_t)w * V + v] = fl[(w - 1) * B];
}

// =============================================================================================
// K-chain: fused pointwise voice chain (+ master-bus tree). Replaces, for every voice at once,
// the executor loop schedule.rs:299-342 over {VolumeProcessor volume.rs:116-143, PanProcessor,
// HardClip hard_clip.rs:70-90, MonoToStereo :46-48, StereoToMono :49-54} and the SumNode tree
// (sum.rs:69-81). Intermediate edges live in registers; HBM sees the input once and either the
// per-voice output or a 1/64-size partial bus.
//
// Mapping: a warp owns kVPW consecutive voices x one 32*VEC-frame tile; a CTA of kWarps warps owns
// kVPC = 64 consecutive voices. All 2*kVPW loads of a thread are issued before first use.
// =============================================================================================
template <int VEC> struct VecT;
template <> struct VecT<4> {
    using type = float4;
    static __device__ __forceinline__ void load(const float* p, float (&x)[4]) { float4 v = __ldcs(reinterpret_cast<const float4*>(p)); x[0] = v.x; x[1] = v.y; x[2] = v.z; x[3] = v.w; }
    static __device__ __forceinline__ void load_ca(const float* p, float (&x)[4]) { float4 v = __ldg(reinterpret_cast<const float4*>(p)); x[0] = v.x; x[1] = v.y; x[2] = v.z; x[3] = v.w; }
    static __device__ __forceinline__ void store(float* p, const float (&x)[4]) { __stcs(reinterpret_cast<float4*>(p), make_float4(x[0], x[1], x[2], x[3])); }
};
template <> struct VecT<1> {
    using type = float;
    static __device__ __forceinline__ void load(const float* p, float (&x)[1]) { x[0] = __ldcs(p); }
    static __device__ __forceinline__ void load_ca(const float* p, float (&x)[1]) { x[0] = __ldg(p); }
    static __device__ __forceinline__ void store(float* p, const float (&x)[1]) { __stcs(p, x[0]); }
};

// the program on one voice's tile, reading record slot kk
template <int VEC>
__device__ __forceinline__ void apply_chain(const ChainArgs& a, uint32_t kk, uint32_t v, uint32_t t_in_block, float (&x)[2][VEC]) {
    const uint32_t V = a.num_voices, F = a.block_frames;
#pragma unroll 1
    for (uint32_t o = 0; o < a.prog.n_ops; ++o) {
        const ChainOp op = a.prog.ops[o];
        switch (op.kind) {
            case OP_GAIN: {  // volume.rs:116-143: out = in * gain[i] (both channels share the curve)
                const uint32_t m = a.rec.mode(kk, (uint32_t)op.sm0, v, V);
                if (m == REC_CLEAR) {
#pragma unroll
                    for (int i = 0; i < VEC; ++i) { x[0][i] = 0.0f; x[1][i] = 0.0f; }
                } else if (m == REC_CONST) {
                    const float g = a.rec.val(kk, op.sm0, v, V);
#pragma unroll
                    for (int i = 0; i < VEC; ++i) { x[0][i] = __fmul_rn(x[0][i], g); x[1][i] = __fmul_rn(x[1][i], g); }
                } else {
                    float g[VEC];
                    VecT<VEC>::load_ca(a.rec.curve(kk, op.sm0, v, V, F) + t_in_block, g);
#pragma unroll
                    for (int i = 0; i < VEC; ++i) { x[0][i] = __fmul_rn(x[0][i], g[i]); x[1][i] = __fmul_rn(x[1][i], g[i]); }
                }
                break;
            }
            case OP_PAN: {
                const uint32_t m0 = a.rec.mode(kk, (uint32_t)op.sm0, v, V), m1 = a.rec.mode(kk, (uint32_t)op.sm1, v, V);
                if (m0 == REC_CLEAR) {
#pragma unroll
                    for (int i = 0; i < VEC; ++i) { x[0][i] = 0.0f; x[1][i] = 0.0f; }
                } else {
                    float gl[VEC], gr[VEC];
                    if (m0 == REC_CURVE) VecT<VEC>::load_ca(a.rec.curve(kk, op.sm0, v, V, F) + t_in_block, gl);
                    else { const float g = a.rec.val(kk, op.sm0, v, V);
#pragma unroll
                        for (int i = 0; i < VEC; ++i) gl[i] = g; }
                    if (m1 == REC_CURVE) VecT<VEC>::load_ca(a.rec.curve(kk, op.sm1, v, V, F) + t_in_block, gr);
                    else { const float g = a.rec.val(kk, op.sm1, v, V);
#pragma unroll
                        for (int i = 0; i < VEC; ++i) gr[i] = g; }
#pragma unroll
                    for (int i = 0; i < VEC; ++i) { x[0][i] = __fmul_rn(x[0][i], gl[i]); x[1][i] = __fmul_rn(x[1][i], gr[i]); }
                }
                break;
            }
            case OP_CLIP: {  // hard_clip.rs:70-76: in.min(t).max(-t)
                const float th = op.f0;
#pragma unroll
                for (int i = 0; i < VEC; ++i) { x[0][i] = fmaxf(fminf(x[0][i], th), -th); x[1][i] = fmaxf(fminf(x[1][i], th), -th); }
                break;
            }
            case OP_M2S:  // mono_to_stereo.rs:46-48
#pragma unroll
                for (int i = 0; i < VEC; ++i) x[1][i] = x[0][i];
                break;
            case OP_S2M:  // stereo_to_mono.rs:49-54: (l + r) * 0.5
#pragma unroll
                for (int i = 0; i < VEC; ++i) x[0][i] = __fmul_rn(__fadd_rn(x[0][i], x[1][i]), 0.5f);
                break;
            default: break;
        }
    }
}

constexpr int kVPC = 64;  // voices per CTA (one partial bus per CTA in the bus variant)

template <int VEC, int CIN, bool BUS, int kVPW, int kWarps, int kMinBlocks>
__global__ void __launch_bounds__(kWarps * 32, kMinBlocks) chain_kernel(ChainArgs a) {
    static_assert(kVPW * kWarps == kVPC, "a CTA owns 64 voices");
    pdl_launch_dependents();
    const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    const uint32_t T = a.frames, V = a.num_voices, F = a.block_frames;
    // Bus variant: CTA slice z sums channels 2z and 2z + 1 of a C-channel bus (C = prog.c_out, up to kMaxBusChannels), an odd last
    // channel alone; the channels are independent trees, so a bus over C channels is ceil(C / 2) stereo reductions on grid.z.
    const uint32_t zc = BUS ? 2u * blockIdx.z : 0u;
    const uint32_t c_out = BUS ? min(2u, a.prog.c_out - zc) : a.prog.c_out;
    constexpr uint32_t kTile = 32u * VEC;
    const uint32_t t = blockIdx.x * kTile + lane * VEC;
    const bool t_ok = t < T;
    const uint32_t vcta = blockIdx.y * kVPC, v0 = vcta + warp * kVPW;
    const uint32_t k = t_ok ? t / F : 0;
    const uint32_t t_in_block = t - k * F;
    // FULL: every voice and every frame of this CTA's tile exists and nothing is zeroed: no bounds checks at all
    const bool full = (vcta + kVPC <= V) && ((blockIdx.x + 1u) * kTile <= T) && !a.zero_first_block;

    // ---- issue every sample load of this thread up front (independent of the control kernel, unless this stage
    //      consumes the output of the preceding kernel) -------------------------------------------------
    if (a.in_from_prev_kernel) pdl_wait();
    float x[kVPW][2][VEC];
    if (full) {
        const float* p[2] = {a.in_ch[zc] + (size_t)v0 * a.in_vstride + t, a.in_ch[zc + CIN - 1] + (size_t)v0 * a.in_vstride + t};
#pragma unroll
        for (int j = 0; j < kVPW; ++j) {
#pragma unroll
            for (int c = 0; c < CIN; ++c) { VecT<VEC>::load(p[c], x[j][c]); p[c] += a.in_vstride; }
            if (CIN == 1) {
#pragma unroll
                for (int i = 0; i < VEC; ++i) x[j][1][i] = 0.0f;
            }
        }
    } else {
        const bool zero_in = a.zero_first_block && k == 0;  // Q11: first block after a schedule swap reads a fresh (zero) pool
#pragma unroll
        for (int j = 0; j < kVPW; ++j) {
            const uint32_t v = v0 + j;
#pragma unroll
            for (int c = 0; c < 2; ++c) {
#pragma unroll
                for (int i = 0; i < VEC; ++i) x[j][c][i] = 0.0f;
                if (c < CIN && t_ok && v < V && !zero_in) VecT<VEC>::load(a.in_ch[zc + (c < CIN ? c : 0)] + (size_t)v * a.in_vstride + t, x[j][c]);
            }
        }
    }

    pdl_wait();  // records written by the control kernel of this call are visible from here on

    // ---- per-warp record staging: one independent load per voice, no CTA-wide barrier ---------------
    // Steady voices (block >= steady_k[v], all smoothers REC_CONST) take the fast path; a warp that owns any
    // transient / CLEAR / CURVE voice, or a tile that straddles block boundaries, takes the generic path.
    // Only the program's own smoothers are staged, at program-local indices.
    __shared__ float s_wv[kWarps][kMaxProgSmoothers][kVPW];
    const bool cta_uniform = (F % kTile) == 0u;
    bool warp_fast = false;
    if (cta_uniform) {
        const uint32_t kb = (blockIdx.x * kTile) / F;
        uint32_t special = 0;
        if (lane < kVPW && v0 + lane < V) special = (kb < a.rec.steady_k[v0 + lane]) || (a.rec.st_modes[v0 + lane] != 0u);
        for (uint32_t i = lane; i < a.prog.n_sm * kVPW; i += 32u) {
            const uint32_t s = i / kVPW, j = i % kVPW;
            s_wv[warp][s][j] = (v0 + j < V) ? a.rec.st_val(a.prog.sm[s], v0 + j, V) : 0.0f;
        }
        warp_fast = !__any_sync(0xffffffffu, special);
        __syncwarp();
    }

    if (warp_fast) {
        // ops outermost (one uniform decode per op), the warp's voices innermost; multipliers are smem broadcasts
#pragma unroll 1
        for (uint32_t o = 0; o < a.prog.n_ops; ++o) {
            const ChainOp op = a.prog.ops[o];
            if (op.kind == OP_GAIN) {  // volume.rs:123-126
#pragma unroll
                for (int j = 0; j < kVPW; ++j) {
                    const float g = s_wv[warp][op.l0][j];
#pragma unroll
                    for (int i = 0; i < VEC; ++i) { x[j][0][i] = __fmul_rn(x[j][0][i], g); x[j][1][i] = __fmul_rn(x[j][1][i], g); }
                }
            } else if (op.kind == OP_PAN) {
#pragma unroll
                for (int j = 0; j < kVPW; ++j) {
                    const float gl = s_wv[warp][op.l0][j], gr = s_wv[warp][op.l1][j];
#pragma unroll
                    for (int i = 0; i < VEC; ++i) { x[j][0][i] = __fmul_rn(x[j][0][i], gl); x[j][1][i] = __fmul_rn(x[j][1][i], gr); }
                }
            } else if (op.kind == OP_CLIP) {  // hard_clip.rs:70-76
                const float th = op.f0;
#pragma unroll
                for (int j = 0; j < kVPW; ++j)
#pragma unroll
                    for (int i = 0; i < VEC; ++i) { x[j][0][i] = fmaxf(fminf(x[j][0][i], th), -th); x[j][1][i] = fmaxf(fminf(x[j][1][i], th), -th); }
            } else if (op.kind == OP_M2S) {  // mono_to_stereo.rs:46-48
#pragma unroll
                for (int j = 0; j < kVPW; ++j)
#pragma unroll
                    for (int i = 0; i < VEC; ++i) x[j][1][i] = x[j][0][i];
            } else if (op.kind == OP_S2M) {  // stereo_to_mono.rs:49-54
#pragma unroll
                for (int j = 0; j < kVPW; ++j)
#pragma unroll
                    for (int i = 0; i < VEC; ++i) x[j][0][i] = __fmul_rn(__fadd_rn(x[j][0][i], x[j][1][i]), 0.5f);
            }
        }
    } else {
        // rare: park the tile in local memory and run the generic per-voice interpreter over it
        float xs[kVPW][2][VEC];
#pragma unroll
        for (int j = 0; j < kVPW; ++j)
#pragma unroll
            for (int c = 0; c < 2; ++c)
#pragma unroll
                for (int i = 0; i < VEC; ++i) xs[j][c][i] = x[j][c][i];
#pragma unroll 1
        for (int j = 0; j < kVPW; ++j) {  // xs is indexed dynamically on purpose: it lives in local memory
            const uint32_t v = v0 + j;
            if (v < V && t_ok) apply_chain<VEC>(a, a.rec.slot(k, v, V), v, t_in_block, xs[j]);
        }
#pragma unroll
        for (int j = 0; j < kVPW; ++j)
#pragma unroll
            for (int c = 0; c < 2; ++c)
#pragma unroll
                for (int i = 0; i < VEC; ++i) x[j][c][i] = xs[j][c][i];
    }

    if (!BUS) {
        if (full) {
            float* q[2] = {a.out_ch[0] + (size_t)v0 * a.out_vstride + t, a.out_ch[1] + (size_t)v0 * a.out_vstride + t};
#pragma unroll
            for (int j = 0; j < kVPW; ++j)
#pragma unroll
                for (int c = 0; c < 2; ++c) if (c < c_out) { VecT<VEC>::store(q[c], x[j][c]); q[c] += a.out_vstride; }
        } else {
#pragma unroll
            for (int j = 0; j < kVPW; ++j) {
                const uint32_t v = v0 + j;
                if (v < V && t_ok) {
#pragma unroll
                    for (int c = 0; c < 2; ++c) if (c < c_out) VecT<VEC>::store(a.out_ch[c] + (size_t)v * a.out_vstride + t, x[j][c]);
                }
            }
        }
    } else {
        // Balanced tree over voices: (2i, 2i+1) per level; a right operand that lies beyond the last voice is
        // skipped (the 1-port SumNode copy, sum.rs:58-65). log2(kVPW) levels in registers per thread.
#pragma unroll
        for (int step = 1; step < kVPW; step <<= 1)
#pragma unroll
            for (int j = 0; j + step < kVPW; j += 2 * step)
                if (full || v0 + j + step < V) {
#pragma unroll
                    for (int c = 0; c < 2; ++c)
#pragma unroll
                        for (int i = 0; i < VEC; ++i) x[j][c][i] = __fadd_rn(x[j][c][i], x[j + step][c][i]);
                }
        // Remaining log2(kWarps) levels through shared memory; each lane owns its own frames. Producer warps
        // arrive on a named barrier and leave; warp c (< c_out, the slice's width) waits, finishes channel zc + c and stores it.
        __shared__ float s_red[kWarps][2][32 * VEC];
#pragma unroll
        for (int c = 0; c < 2; ++c)
#pragma unroll
            for (int i = 0; i < VEC; ++i) s_red[warp][c][lane * VEC + i] = x[0][c][i];
        if (warp >= c_out) { asm volatile("bar.arrive 1, %0;" ::"n"(kWarps * 32) : "memory"); return; }
        asm volatile("bar.sync 1, %0;" ::"n"(kWarps * 32) : "memory");
        if (t_ok) {
            const uint32_t c = warp;
            float p[kWarps][VEC];
#pragma unroll
            for (int w = 0; w < kWarps; ++w)
#pragma unroll
                for (int i = 0; i < VEC; ++i) p[w][i] = s_red[w][c][lane * VEC + i];
#pragma unroll
            for (int step = 1; step < kWarps; step <<= 1)
#pragma unroll
                for (int w = 0; w + step < kWarps; w += 2 * step)
                    if (full || vcta + (w + step) * kVPW < V) {
#pragma unroll
                        for (int i = 0; i < VEC; ++i) p[w][i] = __fadd_rn(p[w][i], p[w + step][i]);
                    }
            VecT<VEC>::store(a.out + ((size_t)blockIdx.y * a.prog.c_out + zc + c) * (a.bus_pitch ? a.bus_pitch : T) + t, p[0]);
        }
    }
}

// K-sum: multi-port SumNode over pool buffers (generic lowering). sum.rs:52-56: all inputs flagged silent -> outputs
// cleared to +0.0 (flagged buffers hold +-0.0, and -0.0 + -0.0 would give -0.0); sum.rs:69-110: ports 2-4 add left to
// right unconditionally; sum.rs:111-133: ports >= 5 start from port 0 and skip ports flagged silent.
template <int VEC>
__global__ void __launch_bounds__(128) sum_kernel(const __grid_constant__ SumArgs a) {
    pdl_launch_dependents();
    pdl_wait();
    const uint32_t t = (blockIdx.y * blockDim.x + threadIdx.x) * VEC, v = blockIdx.x, T = a.frames, V = a.num_voices;  // voices on grid.x (no 65535 cap)
    if (t >= T) return;
    const size_t off = (size_t)v * T + t;
    uint64_t mask = 0;
    if (a.mask_slot >= 0) mask = a.rec.block_in_mask(t / a.block_frames, a.mask_slot, v, V);
    float acc[VEC];
    if (a.mask_slot >= 0 && (mask & a.all_mask) == a.all_mask) {
#pragma unroll
        for (int i = 0; i < VEC; ++i) acc[i] = 0.0f;
        VecT<VEC>::store(a.out + off, acc);
        return;
    }
    VecT<VEC>::load(a.in[0] + off, acc);
    for (uint32_t p = 1; p < a.n_ports; ++p) {
        if (a.skip_silent && ((mask >> a.mask_bit[p]) & 1ull)) continue;
        float x[VEC];
        VecT<VEC>::load(a.in[p] + off, x);
#pragma unroll
        for (int i = 0; i < VEC; ++i) acc[i] = __fadd_rn(acc[i], x[i]);
    }
    VecT<VEC>::store(a.out + off, acc);
}

// K-silence-fix (generic lowering): the reference's non-fused node bodies write +0.0 to an output channel whose input
// channel(s) are flagged silent (volume.rs:131-135, hard_clip.rs:78-82, mono_to_stereo.rs:41-44, stereo_to_mono.rs:41-47)
// where the arithmetic on the flagged +-0.0 samples could give -0.0. Rewrites `out` with +0.0 for every (voice, block)
// whose input mask contains all bits of `test`.
template <int VEC>
__global__ void __launch_bounds__(128) silence_fix_kernel(const __grid_constant__ SilenceFixArgs a) {
    pdl_launch_dependents();
    pdl_wait();
    const uint32_t t = (blockIdx.y * blockDim.x + threadIdx.x) * VEC, v = blockIdx.x, T = a.frames, V = a.num_voices;  // voices on grid.x (no 65535 cap)
    if (t >= T) return;
    const uint64_t mask = a.rec.block_in_mask(t / a.block_frames, a.mask_slot, v, V);
    if ((mask & a.test) != a.test) return;
    float z[VEC];
#pragma unroll
    for (int i = 0; i < VEC; ++i) z[i] = 0.0f;
    VecT<VEC>::store(a.out + (size_t)v * T + t, z);
}

// Dense per-(block, voice) input silence masks of one mask slot, for a custom node's process_device (fw_device_block::in_silence_masks).
__global__ void __launch_bounds__(128) expand_masks_kernel(Records rec, uint32_t mask_slot, uint32_t V, uint32_t n_blocks, uint64_t* __restrict__ out) {
    pdl_launch_dependents();
    pdl_wait();
    const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x, k = blockIdx.y;
    if (v >= V || k >= n_blocks) return;
    Records::at_kv(out, k, v, V) = rec.block_in_mask(k, mask_slot, v, V);
}

// K-sampler: SamplerNode data plane (sampler.rs:445-559 + sample_resource.rs:337-456). One thread = VEC frames of one
// (voice, output channel); what the block plays comes from the control kernel's SmpRec, the samples straight from the
// resource in HBM (converted per sample_resource.rs:337-345), times the node's gain record.
__device__ __forceinline__ float smp_fetch(const ResDesc& d, uint32_t ch, uint64_t pos) {
    if (pos >= d.frames) return 0.0f;  // the reference panics on this slice bound; defined as 0.0 here and in the oracle
    switch (d.fmt) {
        case FW_SAMPLE_F32_PLANAR: return static_cast<const float*>(d.data)[(size_t)ch * d.frames + pos];
        case FW_SAMPLE_F32_INTERLEAVED: return static_cast<const float*>(d.data)[pos * d.channels + ch];
        case FW_SAMPLE_I16_INTERLEAVED: return __fmul_rn((float)static_cast<const int16_t*>(d.data)[pos * d.channels + ch], 1.0f / 32767.0f);
        case FW_SAMPLE_U16_INTERLEAVED: return __fsub_rn(__fmul_rn((float)static_cast<const uint16_t*>(d.data)[pos * d.channels + ch], 2.0f / 65535.0f), 1.0f);
        case FW_SAMPLE_I16_PLANAR: return __fmul_rn((float)static_cast<const int16_t*>(d.data)[(size_t)ch * d.frames + pos], 1.0f / 32767.0f);
        default: return __fsub_rn(__fmul_rn((float)static_cast<const uint16_t*>(d.data)[(size_t)ch * d.frames + pos], 2.0f / 65535.0f), 1.0f);
    }
}
template <int VEC>
__global__ void __launch_bounds__(128) sampler_kernel(const __grid_constant__ SamplerArgs a) {
    pdl_launch_dependents();
    pdl_wait();
    const uint32_t t = (blockIdx.y * blockDim.x + threadIdx.x) * VEC, v = blockIdx.x, c = blockIdx.z, T = a.frames, V = a.num_voices, F = a.block_frames;
    if (t >= T) return;
    const uint32_t k = t / F, f0 = t - k * F;
    const SmpRec r = Records::at_kv(a.srec, k, v, V);
    float y[VEC];
#pragma unroll
    for (int i = 0; i < VEC; ++i) y[i] = 0.0f;
    float* dst = a.out[c] + (size_t)v * a.out_vstride + t;
    if (r.mode == SMP_CLEAR) { VecT<VEC>::store(dst, y); return; }  // clear_all_outputs
    const ResDesc d = a.res_tab[a.res[v] - 1];
    const uint32_t filled = min(a.n_out, d.channels);
    uint32_t src_ch = c;
    if (c >= filled) {
        if (a.n_out == 2 && d.channels == 1) src_ch = 0;              // :546-551 mono sample, stereo node: duplicate
        else { VecT<VEC>::store(dst, y); return; }                    // :552-558 zeroed (and flagged by the control kernel)
    }
    const uint32_t kk = a.rec.slot(k, v, V);
    const uint32_t m = a.rec.mode(kk, (uint32_t)a.sm, v, V);
    float g[VEC];
    if (m == REC_CURVE) {
        const float* curve = a.rec.curve(kk, a.sm, v, V, F) + f0;
#pragma unroll
        for (int i = 0; i < VEC; ++i) g[i] = curve[i];
    } else {
        const float gc = a.rec.val(kk, a.sm, v, V);
#pragma unroll
        for (int i = 0; i < VEC; ++i) g[i] = gc;
    }
    const uint64_t wrap = r.mode == SMP_PLAY_WRAP ? a.loop_start[v] : 0ull;
#pragma unroll
    for (int i = 0; i < VEC; ++i) {
        const uint32_t f = f0 + i;
        float x = 0.0f;  // ZERO_TAIL: frames past the sample's end (:509-511)
        if (f < r.first) x = smp_fetch(d, src_ch, r.p0 + f);
        else if (r.mode == SMP_PLAY_WRAP) x = smp_fetch(d, src_ch, wrap + (f - r.first));
        y[i] = __fmul_rn(x, g[i]);  // :522-543
    }
    VecT<VEC>::store(dst, y);
}

// K-resampler: polyphase windowed-sinc sample player (SURVEY §8 a13, spec in include/fw_b200.h). One thread = one output
// frame of one (voice, channel): the read position is analytic (pos + n * step, Q32.32), so frames are independent.
// Accumulation order (taps ascending, separate multiply and add) matches the oracle bit for bit.
__global__ void resampler_end_kernel(uint64_t* pos, const uint64_t* step, const uint32_t* flags, const uint32_t* res, uint32_t V, uint32_t frames) {
    const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v < V && (flags[v] & 1u) && res[v] != 0) pos[v] += (uint64_t)frames * step[v];
}
__global__ void __launch_bounds__(128) resampler_kernel(const __grid_constant__ ResamplerArgs a) {
    const uint32_t n = blockIdx.y * blockDim.x + threadIdx.x, v = blockIdx.x, c = blockIdx.z;
    if (n >= a.frames) return;
    float* dst = a.out[c] + (size_t)v * a.out_vstride + n;
    const uint32_t r = a.res[v], fl = a.flags[v];
    if (!(fl & 1u) || r == 0) { *dst = 0.0f; return; }
    const ResDesc d = a.res_tab[r - 1];
    uint32_t src_ch = c;
    if (c >= min(a.n_out, d.channels)) {
        if (a.n_out == 2 && d.channels == 1) src_ch = 0;
        else { *dst = 0.0f; return; }
    }
    const uint64_t p = a.pos[v] + (uint64_t)n * a.step[v];
    const int64_t len = (int64_t)d.frames, i0 = (int64_t)(p >> 32) - (int64_t)(a.taps / 2 - 1);
    const float* h = a.table + (size_t)((uint32_t)(p & 0xffffffffull) >> a.phase_shift) * a.taps;
    float y = 0.0f;
    for (uint32_t t = 0; t < a.taps; ++t) {
        int64_t idx = i0 + (int64_t)t;
        float x = 0.0f;
        if (fl & 2u) { idx %= len; if (idx < 0) idx += len; x = smp_fetch(d, src_ch, (uint64_t)idx); }
        else if (idx >= 0 && idx < len) x = smp_fetch(d, src_ch, (uint64_t)idx);
        y = __fadd_rn(y, __fmul_rn(__ldg(h + t), x));
    }
    *dst = y;
}

// K-combine: radix-16 levels of the same balanced tree over partial buses [n_in][rows][T] -> [ceil(n_in/16)][rows][T].
template <int VEC>
__global__ void __launch_bounds__(128) combine_kernel(const float* __restrict__ pin, float* __restrict__ pout, uint32_t n_in, uint32_t rows, uint32_t T, uint32_t out_pitch,
                                                      uint32_t* done_word, uint32_t* done_counter, uint32_t done_epoch) {
    pdl_launch_dependents();
    pdl_wait();  // the partial buses come from the preceding kernel
    const uint32_t t = (blockIdx.x * blockDim.x + threadIdx.x) * VEC;
    const uint32_t row = blockIdx.y, g = blockIdx.z, p0 = g * 16u;
    if (t < T) {
    float p[16][VEC];
#pragma unroll
    for (int j = 0; j < 16; ++j) {
#pragma unroll
        for (int i = 0; i < VEC; ++i) p[j][i] = 0.0f;
        if (p0 + j < n_in) VecT<VEC>::load(pin + ((size_t)(p0 + j) * rows + row) * T + t, p[j]);
    }
#define FW_COMB1(d, s, first)                                                                  \
    if ((first) < n_in) { _Pragma("unroll") for (int i = 0; i < VEC; ++i) p[d][i] = __fadd_rn(p[d][i], p[s][i]); }
#pragma unroll
    for (int step = 1; step < 16; step <<= 1)
#pragma unroll
        for (int j = 0; j + step < 16; j += 2 * step) FW_COMB1(j, j + step, p0 + j + step)
#undef FW_COMB1
    VecT<VEC>::store(pout + ((size_t)g * rows + row) * out_pitch + t, p[0]);
    }
    // Multi-rank hand-over folded into the kernel that completes the rank-local bus (exchange.cu): the last CTA to finish publishes
    // the exchange epoch in a device word the side stream polls — no extra kernel and no event on the main stream's PDL chain.
    if (done_word != nullptr) {
        __threadfence();
        __syncthreads();
        if (threadIdx.x == 0 && atomicAdd(done_counter, 1u) == gridDim.x * gridDim.y * gridDim.z - 1u) {
            *done_counter = 0u;
            __threadfence();
            st_release_gpu(done_word, done_epoch);
        }
    }
}

// =============================================================================================
// Stream boundary: (de)interleave (util.rs:44-147) for the host-facing process_interleaved.
// =============================================================================================
__global__ void deinterleave_kernel(const float* __restrict__ inter, float* __restrict__ planar, uint32_t V, uint32_t C, uint32_t T) {
    const size_t n = (size_t)V * C * T;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const uint32_t f = i % T; const size_t vc = i / T; const uint32_t c = vc % C; const size_t v = vc / C;
        planar[i] = inter[(v * T + f) * C + c];
    }
}
// masks: per-voice graph_out silence masks (or one bus mask when rows_per_mask == 0 is not used: n_masks = 1)
__global__ void interleave_kernel(const float* __restrict__ planar, float* __restrict__ inter, const uint64_t* __restrict__ masks,
                                  uint32_t V, uint32_t C, uint32_t T, uint32_t block_frames) {
    const size_t n = (size_t)V * C * T;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const uint32_t c = i % C; const size_t vf = i / C; const uint32_t f = vf % T; const size_t v = vf / T;
        // The mask handed to interleave is the last block's; silent-flagged buffers hold +0.0 anyway
        // (util.rs:171), so applying it to the final block only is value-identical for earlier blocks.
        const uint64_t m = masks ? masks[v] : 0ull;
        const bool last_block = f >= ((T - 1) / block_frames) * block_frames;
        bool silent;
        if (C == 2) silent = (m & 3ull) == 3ull;            // interleave_stereo util.rs:129-134
        else silent = c < 64 && ((m >> c) & 1ull);           // interleave util.rs:103-107
        inter[i] = (silent && last_block) ? 0.0f : planar[(v * C + c) * T + f];
    }
}

// Ordered small stores (timed parameter commands, plan.hpp PokeArgs): entries are applied one after the other.
__global__ void __launch_bounds__(128) poke_kernel(const __grid_constant__ PokeArgs a) {
    pdl_launch_dependents();
    pdl_wait();
    for (uint32_t i = 0; i < a.n; ++i) {
        uint8_t* base = static_cast<uint8_t*>(a.ptr[i]);
        for (uint32_t j = threadIdx.x; j < a.count[i]; j += blockDim.x) {
            if (a.bytes[i] == 8) *reinterpret_cast<uint64_t*>(base + (size_t)j * a.stride_bytes[i]) = a.val[i];
            else *reinterpret_cast<uint32_t*>(base + (size_t)j * a.stride_bytes[i]) = (uint32_t)a.val[i];
        }
        __syncthreads();
    }
}

__global__ void fill_kernel(float* __restrict__ p, size_t n, float val) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) p[i] = val;
}

// `rows` rows of T frames in each of `groups` groups: row r of group g starts at p + g * group_pitch + r * row_pitch
__global__ void zero_rows_kernel(float* __restrict__ p, uint32_t T, uint64_t row_pitch, uint32_t groups, uint64_t group_pitch) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= T) return;
    for (uint32_t g = blockIdx.z; g < groups; g += gridDim.z) p[g * group_pitch + blockIdx.y * row_pitch + t] = 0.0f;
}

// bus mask: V == 1 -> the voice's mask; else ALL(n_out) iff every voice is all-silent (2-port SumNode tree, sum.rs:52-56)
__global__ void bus_mask_kernel(const uint64_t* __restrict__ gout_mask, uint32_t V, uint32_t n_out, uint64_t* __restrict__ bus_mask) {
    __shared__ int any_audible;
    if (threadIdx.x == 0) any_audible = 0;
    __syncthreads();
    const uint64_t all = all_silent_mask(n_out);
    for (uint32_t v = threadIdx.x; v < V; v += blockDim.x) if ((gout_mask[v] & all) != all) any_audible = 1;
    __syncthreads();
    if (threadIdx.x == 0) *bus_mask = (V == 1) ? gout_mask[0] : (any_audible ? 0ull : all);
}

// =============================================================================================
// launchers
// =============================================================================================
static inline unsigned grid_for(size_t n) { size_t b = (n + 255) / 256; return (unsigned)(b < 132u * 16u ? b : 132u * 16u); }
#define FW_LAUNCH_CHECK() do { cudaError_t e_ = cudaGetLastError(); if (e_ != cudaSuccess) return e_; } while (0)

// The per-call kernels here are launched with programmatic stream serialization (pdl = true): each begins with
// pdl_launch_dependents() and reads its predecessor's results only after pdl_wait().

// 4-wide vectors when both frame counts are multiples of 4 and `addr_bits`, the OR of every address and byte stride the kernel
// steps through, is a multiple of 16
static bool vec4_ok(uint32_t frames, uint32_t block_frames, uintptr_t addr_bits) {
    return frames % 4 == 0 && block_frames % 4 == 0 && addr_bits % 16 == 0;
}

// Threads per CTA of the control kernel: 128 while the shared-memory flags of a voice (two copies of words 1 .. n_flag_words - 1) fit in
// 48 KB for all of them, else fewer, up to the device's opt-in limit; 0 when not even one voice fits.
uint32_t control_threads(uint32_t n_flag_words, int device) {
    const size_t per_thread = 2 * sizeof(uint64_t) * (size_t)(n_flag_words - 1);
    if (per_thread * 128 <= 48 * 1024) return 128;
    int optin = 0;
    if (cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, device) != cudaSuccess) return 0;
    uint32_t t = 64;
    while (t > 0 && per_thread * t > (size_t)optin) t >>= 1;
    return t;
}
cudaError_t launch_control(ControlArgs a, cudaStream_t st) {
    int device = 0;
    cudaGetDevice(&device);
    const CtlTables& tb = a.tables;
    const uint32_t threads = control_threads(tb.n_flag_words, device);
    if (threads == 0) return cudaErrorInvalidValue;
    size_t smem = 2 * sizeof(uint64_t) * (size_t)(tb.n_flag_words - 1) * threads;
    a.stage_tables = smem + tb.image_bytes <= 48 * 1024 ? 1u : 0u;  // larger tables are read from global memory, where L1 keeps them after the first block
    if (a.stage_tables) smem += tb.image_bytes;
    if (smem > 48 * 1024) {
        const cudaError_t e = cudaFuncSetAttribute(control_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
    }
    return launch_ex(control_kernel, dim3((a.num_voices + threads - 1) / threads), dim3(threads), smem, st, true, a);
}

template <int VEC, int CIN, int VPW, int WARPS, int MINB>
static cudaError_t launch_chain_v(const ChainArgs& a, bool bus, cudaStream_t st) {
    dim3 grid((a.frames + 32 * VEC - 1) / (32 * VEC), (a.num_voices + kVPC - 1) / kVPC, bus ? (a.prog.c_out + 1) / 2 : 1);
    if (bus) return launch_ex(chain_kernel<VEC, CIN, true, VPW, WARPS, MINB>, grid, dim3(WARPS * 32), 0, st, true, a);
    return launch_ex(chain_kernel<VEC, CIN, false, VPW, WARPS, MINB>, grid, dim3(WARPS * 32), 0, st, true, a);
}
template <int VEC, int CIN>
static cudaError_t launch_chain_t(const ChainArgs& a, bool bus, cudaStream_t st) {
    if (VEC == 4) return launch_chain_v<VEC, CIN, 4, 16, 2>(a, bus, st);  // 64 regs, 2 x 512 threads per SM
    return launch_chain_v<VEC, CIN, 8, 8, 2>(a, bus, st);
}
cudaError_t launch_chain(const ChainArgs& a, bool bus, cudaStream_t st) {
    uintptr_t al = reinterpret_cast<uintptr_t>(a.out_ch[0]) | reinterpret_cast<uintptr_t>(a.out_ch[1]) | reinterpret_cast<uintptr_t>(a.out) |
                   (uintptr_t)((a.in_vstride | a.out_vstride | a.bus_pitch) * 4);
    for (const float* q : a.in_ch) al |= reinterpret_cast<uintptr_t>(q);
    const bool vec4 = vec4_ok(a.frames, a.block_frames, al);
    if (a.prog.c_in >= 2) return vec4 ? launch_chain_t<4, 2>(a, bus, st) : launch_chain_t<1, 2>(a, bus, st);
    return vec4 ? launch_chain_t<4, 1>(a, bus, st) : launch_chain_t<1, 1>(a, bus, st);
}
uint32_t chain_voice_groups(uint32_t num_voices) { return (num_voices + kVPC - 1) / kVPC; }

cudaError_t launch_combine(const float* pin, float* pout, uint32_t n_in, uint32_t rows, uint32_t T, cudaStream_t st, uint32_t out_pitch,
                           uint32_t* done_word, uint32_t* done_counter, uint32_t done_epoch) {
    if (out_pitch == 0) out_pitch = T;
    // a row of the bus is one block
    const bool vec4 = vec4_ok(T, T, reinterpret_cast<uintptr_t>(pin) | reinterpret_cast<uintptr_t>(pout) | (uintptr_t)out_pitch * 4);
    const uint32_t n_out = (n_in + 15) / 16;
    if (vec4) return launch_ex(combine_kernel<4>, dim3((T / 4 + 127) / 128, rows, n_out), dim3(128), 0, st, true, pin, pout, n_in, rows, T, out_pitch, done_word, done_counter, done_epoch);
    return launch_ex(combine_kernel<1>, dim3((T + 127) / 128, rows, n_out), dim3(128), 0, st, true, pin, pout, n_in, rows, T, out_pitch, done_word, done_counter, done_epoch);
}
cudaError_t launch_sum(const SumArgs& a, cudaStream_t st) {
    uintptr_t al = reinterpret_cast<uintptr_t>(a.out);
    for (uint32_t p = 0; p < a.n_ports; ++p) al |= reinterpret_cast<uintptr_t>(a.in[p]);
    if (vec4_ok(a.frames, a.block_frames, al)) return launch_ex(sum_kernel<4>, dim3(a.num_voices, (a.frames / 4 + 127) / 128), dim3(128), 0, st, true, a);
    return launch_ex(sum_kernel<1>, dim3(a.num_voices, (a.frames + 127) / 128), dim3(128), 0, st, true, a);
}
cudaError_t launch_sampler(const SamplerArgs& a, cudaStream_t st) {
    if (a.n_out == 0 || a.num_voices == 0 || a.frames == 0) return cudaSuccess;
    uintptr_t al = (uintptr_t)(a.out_vstride * 4);
    for (uint32_t c = 0; c < a.n_out; ++c) al |= reinterpret_cast<uintptr_t>(a.out[c]);
    if (vec4_ok(a.frames, a.block_frames, al)) return launch_ex(sampler_kernel<4>, dim3(a.num_voices, (a.frames / 4 + 127) / 128, a.n_out), dim3(128), 0, st, true, a);
    return launch_ex(sampler_kernel<1>, dim3(a.num_voices, (a.frames + 127) / 128, a.n_out), dim3(128), 0, st, true, a);
}
cudaError_t launch_resampler(const ResamplerArgs& a, uint64_t* pos, cudaStream_t st) {
    if (a.n_out && a.num_voices && a.frames) {
        resampler_kernel<<<dim3(a.num_voices, (a.frames + 127) / 128, a.n_out), 128, 0, st>>>(a);
        resampler_end_kernel<<<(a.num_voices + 127) / 128, 128, 0, st>>>(pos, a.step, a.flags, a.res, a.num_voices, a.frames);
    }
    return cudaGetLastError();
}
cudaError_t launch_silence_fix(const SilenceFixArgs& a, cudaStream_t st) {
    if (vec4_ok(a.frames, a.block_frames, reinterpret_cast<uintptr_t>(a.out))) return launch_ex(silence_fix_kernel<4>, dim3(a.num_voices, (a.frames / 4 + 127) / 128), dim3(128), 0, st, true, a);
    return launch_ex(silence_fix_kernel<1>, dim3(a.num_voices, (a.frames + 127) / 128), dim3(128), 0, st, true, a);
}
cudaError_t launch_expand_masks(const Records& rec, uint32_t mask_slot, uint32_t V, uint32_t n_blocks, uint64_t* out, cudaStream_t st) {
    if (V == 0 || n_blocks == 0) return cudaSuccess;
    return launch_ex(expand_masks_kernel, dim3((V + 127) / 128, n_blocks), dim3(128), 0, st, true, rec, mask_slot, V, n_blocks, out);
}
cudaError_t launch_poke(const PokeArgs& a, cudaStream_t st) {
    if (a.n == 0) return cudaSuccess;
    return launch_ex(poke_kernel, dim3(1), dim3(128), 0, st, true, a);
}
cudaError_t launch_deinterleave(const float* inter, float* planar, uint32_t V, uint32_t C, uint32_t T, cudaStream_t st) {
    const size_t n = (size_t)V * C * T; if (n == 0) return cudaSuccess;
    deinterleave_kernel<<<grid_for(n), 256, 0, st>>>(inter, planar, V, C, T);
    return cudaGetLastError();
}
cudaError_t launch_interleave(const float* planar, float* inter, const uint64_t* masks, uint32_t V, uint32_t C, uint32_t T, uint32_t block_frames, cudaStream_t st) {
    const size_t n = (size_t)V * C * T; if (n == 0) return cudaSuccess;
    interleave_kernel<<<grid_for(n), 256, 0, st>>>(planar, inter, masks, V, C, T, block_frames);
    return cudaGetLastError();
}
cudaError_t launch_fill(float* p, size_t n, float val, cudaStream_t st) {
    if (n == 0) return cudaSuccess;
    fill_kernel<<<grid_for(n), 256, 0, st>>>(p, n, val);
    return cudaGetLastError();
}
cudaError_t launch_zero_rows(float* p, uint32_t T, uint64_t row_pitch, uint32_t rows, uint32_t groups, uint64_t group_pitch, cudaStream_t st) {
    if (T == 0 || rows == 0 || groups == 0) return cudaSuccess;
    zero_rows_kernel<<<dim3((T + 255) / 256, rows, std::min(groups, 65535u)), 256, 0, st>>>(p, T, row_pitch, groups, group_pitch);
    return cudaGetLastError();
}
cudaError_t launch_bus_mask(const uint64_t* gout_mask, uint32_t V, uint32_t n_out, uint64_t* bus_mask, cudaStream_t st) {
    bus_mask_kernel<<<1, 256, 0, st>>>(gout_mask, V, n_out, bus_mask);
    return cudaGetLastError();
}

}  // namespace fw
