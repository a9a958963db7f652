// plan.hpp — PODs shared by the host lowering and the sm_90a kernels.
//
// A compiled voice graph is lowered to
//   * CtlTables  — the schedule as the CONTROL kernel sees it (device arrays built once per plan): one thread per
//                  voice walks the scheduled nodes per block and restates the reference's per-block control logic
//                  (silence flags schedule.rs:305-341, ParamSmoother state machine smoother.rs:115-194,
//                  gain's early-outs volume.rs:94-108), emitting one small record per (voice, block);
//   * ChainProgram — the DATA plane: a linear chain of pointwise node bodies fused into one
//                  streaming kernel, optionally ending in the master-bus tree sum.
#pragma once
#include <cstdint>

namespace fw {

constexpr int kMaxChainOps = 16;
constexpr int kMaxProgSmoothers = 16;  // distinct smoothers one ChainProgram reads (the chain kernel stages them in shared memory)
constexpr int kModesPerWord = 16;      // 2 mode bits per smoother in a 32-bit record word

constexpr int kMaxBusChannels = 8;  // graph_out channels of a master bus (7.1, the most an HDMI LPCM output carries); FW_MAX_BUS_CHANNELS

enum SmStatus : uint32_t { SM_INACTIVE = 0, SM_ACTIVE = 1, SM_DEACTIVATING = 2 };   // smoother.rs:29-39
enum RecMode : uint32_t { REC_CONST = 0, REC_CLEAR = 1, REC_CURVE = 2 };

enum ChainOpKind : uint32_t { OP_GAIN = 0, OP_PAN = 1, OP_CLIP = 2, OP_M2S = 3, OP_S2M = 4 };
// sm0 / sm1: the plan's smoother indices (-1: none); l0 / l1: the same smoothers' program-local indices (ChainProgram::sm[l] = sm),
// where the chain kernel stages the steady values
struct ChainOp { uint32_t kind; int32_t sm0, sm1; float f0; int32_t l0, l1; };
struct ChainProgram { uint32_t n_ops, c_in, c_out, n_sm; ChainOp ops[kMaxChainOps]; int32_t sm[kMaxProgSmoothers]; };

struct CtlNode {
    uint8_t kind, n_in, n_out, pad;
    uint32_t in_off, out_off;   // into CtlTables::in_port / out_port
    int32_t sm0, sm1;           // smoother indices (-1: none); SamplerNode / ResamplerNode: sm1 = index into CtlTables::smp / rs; custom node: sm0 = fw_out_silence_rule
    uint32_t mask_slot;         // 1 + mask slot of Records::in_masks, 0 = none
};
// One smoother: its per-voice state (SoA over voices, owned by the node's device state) and its target parameter
struct SmDesc { float* input; float* last; uint32_t* status; const float* target; };

// ---- SamplerNode (sampler.rs:283-560) on the device ----
// Sample resources (sample_resource.rs): one descriptor per uploaded resource; handles are index + 1.
struct ResDesc { const void* data; uint64_t frames; uint32_t channels, fmt; };  // fmt: fw_sample_format
// NodeToProcessorMsg (sampler.rs:21-28) with seconds already converted to frames on the host (pure f64 arithmetic)
enum SmpMsgKind : uint32_t { SMSG_SET_SAMPLE = 0, SMSG_PLAY = 1, SMSG_PAUSE = 2, SMSG_STOP = 3, SMSG_SET_PLAYHEAD = 4, SMSG_SET_LOOP = 5 };
struct SamplerMsgDev { uint32_t kind, a; uint64_t x, y; };  // SET_SAMPLE: a = handle, x = stop_playback; SET_PLAYHEAD: x = frame; SET_LOOP: a = fw_loop_mode, x = start, y = end
// What one block of one voice plays: frames [0, first) come from resource frames p0.., the rest from the loop start
// (WRAP), or is zero (ZERO_TAIL, the sample ended), sampler.rs:445-516. CLEAR: clear_all_outputs.
enum SmpMode : uint32_t { SMP_CLEAR = 0, SMP_PLAY = 1, SMP_PLAY_WRAP = 2, SMP_PLAY_ZERO_TAIL = 3 };
struct SmpRec { uint64_t p0; uint32_t first, mode; };
// Every sampler and resampler of a context reads the same resource table; each chunk takes one snapshot of it (table and count), which
// the control, sampler and resampler kernels of the chunk all read.
struct RsCtl { const uint32_t* flags; const uint32_t* res; uint32_t n_out, pad; };  // flags: bit0 playing, bit1 loop
struct SamplerCtl {
    // per-voice processor state (SamplerProcessor fields sampler.rs:283-297), persistent across calls
    uint32_t* playing; uint64_t* playhead; uint32_t* loop_flags;  // bit0: loop_range.is_some(), bit1: full_range
    uint64_t* loop_start; uint64_t* loop_end; uint32_t* res;      // res: resource handle, 0 = None
    const SamplerMsgDev* msgs; const uint32_t* msg_off;           // the chunk's messages of voice v: [msg_off[v], msg_off[v+1])
    SmpRec* rec;                                                   // [block][voice]
    uint32_t* last_play;                                           // [voice]: the last block the walk processed played (scratch)
    uint32_t n_out, pad;
};
// The schedule as the control kernel reads it: arrays of the plan, laid out one after the other (each 16-byte aligned) in one device
// buffer, `image`, uploaded once when the graph is lowered; o_*: their byte offsets in it.
//   nodes     CtlNode per scheduled node
//   in_port   per input port: pool buffer | kPortClear when the port is unconnected (schedule.rs:310-313)
//   out_port  per output port: pool buffer
//   sm, smp, rs  SmDesc per smoother, SamplerCtl per SamplerNode, RsCtl per ResamplerNode
struct CtlTables {
    const void* image; uint32_t image_bytes, pad;
    uint32_t o_nodes, o_in_port, o_out_port, o_sm, o_smp, o_rs;
    uint32_t n_nodes, n_smoothers, n_buffers, n_flag_words;  // n_flag_words = ceil(n_buffers / 64)
    uint32_t n_samplers, n_resamplers, n_in_ports, n_out_ports;
};
constexpr uint32_t kCtlParamImage = 2048;  // a table image up to this size also travels in the control kernel's parameters
constexpr uint32_t kPortClear = 0x80000000u;

// Per-call record buffers written by the control kernel, read by the data kernels. k: record slot (kt_max of them), V voices.
//   modes[k][w][v]       2 bits per smoother: smoother s in word w = s / 16, bits 2 (s % 16) (n_mode_words = max(1, ceil(NS / 16)))
//   vals[k][s][v]        constant value of smoother s in block k (REC_CONST)
//   curves[k][s][v][F]   gain curve (REC_CURVE)
//   in_masks[k][m][v]    input silence mask of the node with mask slot m (CtlNode::mask_slot - 1): SumNodes, the silence fix, custom nodes
//   steady_k[v]          blocks >= steady_k[v] reuse the record of block steady_k[v]
//   st_modes[v]          OR of the steady record's mode words: 0 iff every smoother is REC_CONST there (the chain kernel's fast path)
//   st_vals[s][v]        the steady record's constant values, flattened so the data kernels reach them with one independent load
//   st_in_masks[m][v]    the steady record's input masks
// Every index into these buffers, into slot_of and into the samplers' SmpRec arrays is one of the accessors below. Indices are
// widened to 64 bits before they are multiplied.
struct Records {
    uint32_t* modes; float* vals; float* curves; uint32_t* steady_k; uint64_t* gout_mask; uint32_t* error;
    uint32_t* st_modes; float* st_vals;
    uint64_t* in_masks; uint64_t* st_in_masks;
    uint32_t n_mask_slots, n_mode_words;
    uint32_t kt_max, n_smoothers;
    // Graphs with SamplerNodes: a sample that ends mid-call starts a new transient, so "record of block k" is no longer
    // min(k, steady_k): slot_of[k][v] names the record slot explicitly (null for graphs without samplers). steady_k[v] is
    // then the first block of the FINAL steady phase, and st_modes / st_vals its record, so the chain kernel's fast path
    // still applies.
    uint16_t* slot_of;

    // [block][voice] arrays: slot_of, the samplers' SmpRec records, the custom nodes' dense masks
    template <class T> __host__ __device__ static T& at_kv(T* p, uint32_t k, uint32_t v, uint32_t V) { return p[(size_t)k * V + v]; }
    // record slot of block k of voice v
    __host__ __device__ uint32_t slot(uint32_t k, uint32_t v, uint32_t V) const {
        if (slot_of != nullptr) return at_kv(slot_of, k, v, V);
        return min(k, steady_k[v]);
    }
    // word w of the mode bits of record slot kk, and the mode of smoother s there
    __host__ __device__ uint32_t& mode_word(uint32_t kk, uint32_t w, uint32_t v, uint32_t V) const {
        return (modes + (size_t)kk * n_mode_words * V + v)[(size_t)w * V];
    }
    __host__ __device__ uint32_t mode(uint32_t kk, uint32_t s, uint32_t v, uint32_t V) const {
        return (mode_word(kk, s / kModesPerWord, v, V) >> (2 * (s % kModesPerWord))) & 3u;
    }
    __host__ __device__ float& val(uint32_t kk, int32_t s, uint32_t v, uint32_t V) const { return vals[((size_t)kk * n_smoothers + s) * V + v]; }
    __host__ __device__ float& st_val(int32_t s, uint32_t v, uint32_t V) const { return st_vals[(size_t)s * V + v]; }
    __host__ __device__ float* curve(uint32_t kk, int32_t s, uint32_t v, uint32_t V, uint32_t F) const {
        return curves + (((size_t)kk * n_smoothers + s) * V + v) * F;
    }
    __host__ __device__ uint64_t& in_mask(uint32_t kk, uint32_t m, uint32_t v, uint32_t V) const { return in_masks[((size_t)kk * n_mask_slots + m) * V + v]; }
    __host__ __device__ uint64_t& st_in_mask(uint32_t m, uint32_t v, uint32_t V) const { return st_in_masks[(size_t)m * V + v]; }
    // input mask of mask slot m in block k: the steady record's from steady_k on
    __host__ __device__ uint64_t block_in_mask(uint32_t k, uint32_t m, uint32_t v, uint32_t V) const {
        return k >= steady_k[v] ? st_in_mask(m, v, V) : in_mask(slot(k, v, V), m, v, V);
    }

    // element counts of the buffers for V voices and F frames per block (buffers indexed by smoother or mask slot get at least one row)
    size_t modes_count(uint32_t V) const { return (size_t)kt_max * n_mode_words * V; }
    size_t vals_count(uint32_t V) const { return (size_t)kt_max * st_vals_count(V); }
    size_t curves_count(uint32_t V, uint32_t F) const { return (size_t)kt_max * n_smoothers * V * F; }
    size_t st_vals_count(uint32_t V) const { return (size_t)(n_smoothers ? n_smoothers : 1) * V; }
    size_t in_masks_count(uint32_t V) const { return (size_t)kt_max * st_in_masks_count(V); }
    size_t st_in_masks_count(uint32_t V) const { return (size_t)(n_mask_slots ? n_mask_slots : 1) * V; }
    static size_t kv_count(uint32_t K, uint32_t V) { return (size_t)K * V; }
};

// SamplerNode data plane: out[c] + v * out_vstride is channel c of voice v ([T] floats).
struct SamplerArgs {
    float* out[64]; uint64_t out_vstride;
    uint32_t n_out, num_voices, frames, block_frames;
    const SmpRec* srec; const uint32_t* res; const uint64_t* loop_start; const ResDesc* res_tab;
    int32_t sm, pad;   // the node's gain smoother
    Records rec;
};

// Ordered small stores into device arrays (timed parameter commands): entry i writes `count` elements of 4 or 8 bytes.
struct PokeArgs { void* ptr[16]; uint64_t val[16]; uint32_t count[16], stride_bytes[16]; uint8_t bytes[16]; uint32_t n; };

struct ControlArgs {
    CtlTables tables;
    Records rec;
    uint64_t* flags;       // [n_flag_words][V] buffer_silence_flags bitset (schedule.rs:170), persists across calls
    const ResDesc* res_tab; uint32_t n_res;  // the chunk's snapshot of the resource table
    uint32_t smp_msgs;     // some sampler has messages in this chunk (else every msg_off is all zero)
    uint32_t stage_tables; // set by launch_control: each CTA copies the table image to shared memory first
    uint32_t num_voices, frames, block_frames;
    float a, b, eps;       // smoother.rs:99-100,22
    uint32_t err_value;    // written to *rec.error on a record-budget overflow: (call epoch << 4) | 1
    uint32_t image_in_param;  // `image` holds a copy of tables.image (small graphs: read with the launch, not from memory)
    alignas(16) unsigned char image[kCtlParamImage];
};

struct ChainArgs {
    // Channel c of voice v starts at in_ch[c] + v * in_vstride (floats). A staged chain reads [V][c_in][T]
    // (in_ch[c] = base + c*T, in_vstride = c_in*T); the generic lowering reads pool buffers [V][T] (in_vstride = T).
    // Only the bus variant reads more than two channels (in_ch[c_in] repeats an odd last channel); it writes no out_ch.
    const float* in_ch[kMaxBusChannels]; float* out_ch[2];
    uint64_t in_vstride, out_vstride;
    float* out;            // bus variant only: partial bus [G][c_out][bus_pitch]
    uint32_t bus_pitch, pad3;  // floats between the rows of `out` (0: frames); the caller's bus is a column window of longer rows when a call is chunked
    uint32_t num_voices, frames, block_frames, zero_first_block;
    uint32_t in_from_prev_kernel, pad0, pad1, pad2;  // `in` is produced by the preceding kernel: wait before the loads
    Records rec;
    ChainProgram prog;
};

// One pass of the temporal kernel over R = voices * channels rows of T frames.
struct TemporalArgs {
    const float* in; float* out;   // [R][in_pitch] / [R][out_pitch], T frames used
    uint32_t R, C, T, zero_first;  // zero_first: leading frames read as 0.0 (Q11)
    uint32_t ns; const float* coeffs;  // biquad: [R / C][ns][5] = {b0,b1,b2,a1,a2}; ns == 0: no biquad
    float* state;                  // [R][8][2] = {s1, s2}
    uint32_t D; float* ring; uint32_t pos;  // delay: ring [R][D], D == 0: no delay
    uint32_t srow_mul, srow_add;   // state / ring row of data row r = r * srow_mul + srow_add (1, 0 for [V][C][T] input)
    uint32_t svf;                  // 1: `coeffs` holds SVF stages [R / C][ns][6] and the recurrence is the SVF's
    uint32_t row_base;             // lanes kernel: first row of CTA 0 (the ragged last CTA is launched on its own)
    uint32_t in_pitch, out_pitch;  // floats between rows of `in` / `out` (0: T). A call chunk is a column window of longer rows.
    // Two row segments in one pass (generic lowering: two channels of a node live in two pool buffers): rows >= seg_rows read in2 / write out2
    // at row (r - seg_rows) and use state row + 1 (the next channel). seg_rows == 0: one segment.
    const float* in2; float* out2; uint32_t seg_rows, pad_seg;
};

// One call of the FIR reverb (reverb.cu): history roll + bf16 conversion, then the wgmma GEMM.
struct ReverbCall {
    const float* in; float* out;        // [V][C][T] f32
    void* xh;                           // bf16 sample history [C*V][pitch]; the call's block is appended at column `cursor`
    const void* bt;                     // bf16 Toeplitz expansion of the IR [ir_ch][256][kpad]
    uint32_t V, C, T, L, ir_ch, cursor, pitch, zero_first;
    uint32_t chan_base;                 // history rows / IR channel of data channel c are (chan_base + c)
    uint32_t in_pitch, out_pitch;       // floats between (voice, channel) rows of in / out (0: T)
    float* ws; uint32_t* flags; uint32_t epoch;  // tail-wave fix-up of the GEMM: reverb_ws_bytes(), one flag per SM, a launch counter (> 0, unique per launch)
};

// Multi-port SumNode on pool buffers (sum.rs:69-133): out = in[0] + in[1] + ... strictly left to right.
struct SumArgs {
    const float* in[64]; float* out;   // rows [V][T]
    uint8_t mask_bit[64];              // input index (port * n_out + ch) of in[p] inside the node's silence mask
    uint32_t n_ports, num_voices, frames, block_frames;
    int32_t mask_slot;                 // mask slot of Records::in_masks
    uint32_t skip_silent;              // ports >= 5: silent ports are skipped (sum.rs:118-131)
    uint64_t all_mask;                 // all node inputs: every bit set -> outputs cleared (sum.rs:52-56)
    Records rec;
};

// Rewrite one pool buffer with +0.0 wherever the node's input silence mask contains `test` (see silence_fix_kernel).
struct SilenceFixArgs {
    float* out; uint64_t test;
    uint32_t num_voices, frames, block_frames; int32_t mask_slot;
    Records rec;
};

// Polyphase resampler data plane (spec in include/fw_b200.h). out[c] + v * out_vstride is channel c of voice v.
struct ResamplerArgs {
    float* out[64]; uint64_t out_vstride;
    uint32_t n_out, num_voices, frames, taps;
    uint32_t phase_shift, pad;
    const float* table; const uint64_t* pos; const uint64_t* step; const uint32_t* flags; const uint32_t* res; const ResDesc* res_tab;
};

}  // namespace fw
