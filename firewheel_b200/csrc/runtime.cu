// runtime.cu — product runtime behind include/fw_b200.h.
//
//   fw_ctx        main-thread side (FirewheelGraphCtx context.rs:29): graph edits, parameter stores,
//                 compile + lowering + device allocation in update(), plan hand-off.
//   fw_processor  stream side (FirewheelProcessor processor.rs:18): adopts plans from the ring, drains the command
//                 ring, enqueues the control + data kernels on its CUDA stream. It never allocates: per-call
//                 scratch belongs to the plan, I/O staging is sized at activate for max_call_frames.
//   Plan          ScheduleHeapData analogue (schedule.rs:128-150): schedule + device tables + record buffers.
//   NodeDeviceState  the device-resident "processor counterpart" of a node (Box<dyn AudioNodeProcessor>):
//                 parameter mirrors and per-voice state; survives schedule swaps like processors do
//                 (processor.rs:176-197) and is released on the main thread (graph.rs:644-669).
//
// There is no CPU fallback anywhere in this file: without a CUDA device activate() fails.
#include <cuda_runtime.h>
#include <dlfcn.h>

#include <algorithm>
#include <atomic>
#include <chrono>
#include <condition_variable>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "../../include/fw_b200.h"
#include "graph.hpp"
#include "kernels.cuh"
#include "plan.hpp"

namespace fw {

// Last device-side error text. Written on the thread that hit the error (main thread, stream thread, or the fw_stream producer);
// fw_last_device_error() returns the calling thread's own message if it has one, else the most recent one from any thread.
static thread_local std::string g_dev_err;
static std::mutex g_err_mu;              // error path only: never taken on a successful call
static std::string g_err_any;
static void publish_error() { std::lock_guard<std::mutex> lk(g_err_mu); g_err_any = g_dev_err; }
static bool cuda_ok(cudaError_t e, const char* what) {
    if (e == cudaSuccess) return true;
    g_dev_err = std::string(what) + ": " + cudaGetErrorString(e);
    publish_error();
    return false;
}
#define FW_CUDA(call) fw::cuda_ok((call), #call)

// Owner of the device and pinned host memory of one runtime object (ResTable, NodeDeviceState, Plan, fw_processor): everything it
// hands out is freed, on its device, when it is destroyed. The objects keep plain pointers, which travel by value in the kernel
// arguments. ok() turns false for good at the first failed allocation or zero fill, so a run of allocations is checked once.
class DevMem {
  public:
    const int device;
    explicit DevMem(int dev) : device(dev) {}
    DevMem(const DevMem&) = delete; DevMem& operator=(const DevMem&) = delete;
    ~DevMem() { cudaSetDevice(device); for (void* q : dev_) cudaFree(q); for (void* q : host_) cudaFreeHost(q); }
    bool ok() const { return ok_; }
    // n elements (at least one), zero-filled unless `zero` is false
    template <class T> T* dev(size_t n, bool zero = true) {
        void* p = nullptr;
        if (n == 0) n = 1;
        if (!FW_CUDA(cudaMalloc(&p, n * sizeof(T)))) return failed();
        dev_.push_back(p);
        if (zero && !FW_CUDA(cudaMemset(p, 0, n * sizeof(T)))) return failed();
        return static_cast<T*>(p);
    }
    template <class T> T* host(size_t n) {
        void* p = nullptr;
        if (!FW_CUDA(cudaMallocHost(&p, n * sizeof(T)))) return failed();
        host_.push_back(p);
        return static_cast<T*>(p);
    }
  private:
    // the message stays in g_dev_err; the runtime's pending error is cleared so that the next launch check does not report it
    std::nullptr_t failed() { cudaGetLastError(); ok_ = false; return nullptr; }
    std::vector<void*> dev_, host_; bool ok_ = true;
};

// wait-free SPSC ring (rtrb::RingBuffer, context.rs:61-64) of a capacity chosen at construction
template <class T> struct DynSpsc {
    std::unique_ptr<T[]> slots; size_t n = 0;  // n = capacity + 1
    std::atomic<size_t> head{0}, tail{0};
    explicit DynSpsc(size_t capacity) : slots(new T[capacity + 1]), n(capacity + 1) {}
    size_t capacity() const { return n - 1; }
    bool push(const T& v) {
        const size_t t = tail.load(std::memory_order_relaxed), nx = t + 1 == n ? 0 : t + 1;
        if (nx == head.load(std::memory_order_acquire)) return false;
        slots[t] = v; tail.store(nx, std::memory_order_release); return true;
    }
    bool pop(T* out) {
        const size_t h = head.load(std::memory_order_relaxed);
        if (h == tail.load(std::memory_order_acquire)) return false;
        *out = slots[h]; head.store(h + 1 == n ? 0 : h + 1, std::memory_order_release); return true;
    }
};

// Sample resources of one context ("Arc<dyn SampleResource>", sample_resource.rs): uploaded once, referenced by handle.
struct ResTable {
    std::mutex mu;
    DevMem mem;  // the device copies of the sample data and every device table (old ones stay valid for in-flight calls)
    std::vector<ResDesc> host; ResDesc* d_tab = nullptr;  // descriptors and their device table (re-built on every add)
    explicit ResTable(int device) : mem(device) {}
    uint32_t add(uint32_t fmt, uint32_t channels, uint64_t frames, const void* data) {
        const size_t bytes = (size_t)channels * frames * (fmt <= FW_SAMPLE_F32_INTERLEAVED ? 4 : 2);
        cudaSetDevice(mem.device);
        uint8_t* d;
        { std::lock_guard<std::mutex> lk(mu); d = mem.dev<uint8_t>(bytes, false); }  // the upload below runs outside the lock
        if (!d || !FW_CUDA(cudaMemcpy(d, data, bytes, cudaMemcpyHostToDevice))) return 0;
        std::lock_guard<std::mutex> lk(mu);
        host.push_back(ResDesc{d, frames, channels, fmt});
        ResDesc* nt = mem.dev<ResDesc>(host.size(), false);
        if (!nt || !FW_CUDA(cudaMemcpy(nt, host.data(), sizeof(ResDesc) * host.size(), cudaMemcpyHostToDevice))) { host.pop_back(); return 0; }
        d_tab = nt;
        return (uint32_t)host.size();
    }
    void snapshot(const ResDesc** tab, uint32_t* n) { std::lock_guard<std::mutex> lk(mu); *tab = d_tab; *n = (uint32_t)host.size(); }
    bool frames_of(uint32_t handle, uint64_t* frames) { std::lock_guard<std::mutex> lk(mu); if (handle == 0 || handle > host.size()) return false; *frames = host[handle - 1].frames; return true; }
};

struct NodeDeviceState {
    DevMem mem;  // every buffer below
    uint32_t kind = 0, V = 0, n_sm = 0;
    std::shared_ptr<NodeParams> params;
    float* d_target[2] = {nullptr, nullptr};      // the smoothed parameters' targets (NodeKind::target)
    float* sm_input[2] = {nullptr, nullptr};
    float* sm_last[2] = {nullptr, nullptr};
    uint32_t* sm_status[2] = {nullptr, nullptr};
    // temporal nodes: `channels` rows per voice
    uint32_t channels = 0;
    float* d_coeffs = nullptr;   // biquad / SVF [V][ns][coeff_width(kind)]
    float* d_state = nullptr;    // biquad [V*channels][8][2]
    float* d_ring = nullptr;     // delay  [V*channels][D]
    uint32_t ring_pos = 0;       // stream-side cursor into the ring
    // conv reverb: Toeplitz-expanded IR and the ping-pong bf16 sample history (reverb.cu)
    void* d_bt = nullptr; void* d_xh[2] = {nullptr, nullptr}; uint32_t xh_cur = 0, xh_cursor = 0, xh_pitch = 0;  // cursor: where the next block is appended
    float* d_rv_ws = nullptr; uint32_t* d_rv_flags = nullptr; uint32_t rv_epoch = 0;  // tail-wave fix-up of the GEMM (reverb.cu)
    static constexpr uint32_t kReverbMaxFrames = 65536;  // longest call the history buffers are sized for
    // polyphase resampler: table + per-voice transport mirrors + the device-resident Q32.32 position
    float* d_rs_table = nullptr; uint32_t* d_rs_res = nullptr; uint32_t* d_rs_flags = nullptr; uint64_t* d_rs_step = nullptr;
    uint64_t* d_rs_pos = nullptr;
    // sampler: per-voice SamplerProcessor state (sampler.rs:283-297) + this chunk's messages
    uint32_t* d_playing = nullptr; uint64_t* d_playhead = nullptr; uint32_t* d_loop_flags = nullptr; uint64_t* d_loop_start = nullptr; uint64_t* d_loop_end = nullptr; uint32_t* d_res = nullptr;
    SamplerMsgDev* d_msgs = nullptr; size_t cap_msgs = 0; uint32_t* d_msg_off = nullptr; uint32_t cur_n_msgs = 0;  // this chunk's messages on the device
    bool msg_off_dirty = false;  // d_msg_off still holds the offsets of an earlier chunk's messages
    // custom node (plugin vtable): the processor returned by activate() and the dense per-(block, voice) input masks handed to it
    void* custom_proc = nullptr; bool custom_deactivate = false;  // true: released through deactivate(node, processor) (graph.rs:603-609,644-648)
    explicit NodeDeviceState(int device) : mem(device) {}
    ~NodeDeviceState() {  // the plugin lets go of its processor before `mem` frees the node's buffers
        cudaSetDevice(mem.device);
        if (params && params->custom && custom_proc) {  // main thread: plans are released in ctx_drain / ctx_free
            const fw_node_vtable& vt = params->custom->vt;
            if (custom_deactivate && vt.deactivate) vt.deactivate(params->custom->node, custom_proc);
            else if (vt.drop_processor) vt.drop_processor(custom_proc);
        }
        if (ev_staged) cudaEventDestroy(ev_staged);
    }
    // ParamSmoother::new(val): input = last_output = val, Inactive (smoother.rs:93-112; volume.rs:67-75)
    bool create() {
        const NodeKind& nk = node_kind(kind);
        n_sm = nk.target[1] ? 2 : nk.target[0] ? 1 : 0;
        for (uint32_t i = 0; i < n_sm; ++i) {
            d_target[i] = mem.dev<float>(V); sm_input[i] = mem.dev<float>(V); sm_last[i] = mem.dev<float>(V); sm_status[i] = mem.dev<uint32_t>(V);
            if (!mem.ok()) return false;
            const float* h = ((*params).*nk.target[i]).data();
            if (!FW_CUDA(cudaMemcpy(d_target[i], h, V * 4, cudaMemcpyHostToDevice))) return false;
            if (!FW_CUDA(cudaMemcpy(sm_input[i], h, V * 4, cudaMemcpyHostToDevice))) return false;
            if (!FW_CUDA(cudaMemcpy(sm_last[i], h, V * 4, cudaMemcpyHostToDevice))) return false;
        }
        if (const uint32_t w = coeff_width(kind)) {  // biquad / SVF
            d_coeffs = mem.dev<float>((size_t)V * params->num_stages * w, false);
            d_state = mem.dev<float>((size_t)V * channels * 8 * 2);  // zero state
            if (!mem.ok()) return false;
            if (params->num_stages && !FW_CUDA(cudaMemcpy(d_coeffs, params->coeffs.data(), params->coeffs.size() * 4, cudaMemcpyHostToDevice))) return false;
        } else if (kind == FW_NODE_DELAY && params->delay) {
            d_ring = mem.dev<float>((size_t)V * channels * params->delay);  // zero-initialised ring
            if (!mem.ok()) return false;
        } else if (kind == FW_NODE_CONV_REVERB) {
            const uint32_t L = params->ir_len, ich = params->ir_channels, kpad = reverb_kpad(L);
            xh_pitch = reverb_hist(L) + kReverbMaxFrames; xh_cursor = reverb_hist(L);
            d_bt = mem.dev<uint16_t>((size_t)ich * 256 * kpad, false);
            d_xh[0] = mem.dev<uint16_t>((size_t)V * channels * xh_pitch);  // zero history
            d_xh[1] = mem.dev<uint16_t>((size_t)V * channels * xh_pitch);
            d_rv_ws = mem.dev<float>(reverb_ws_bytes() / sizeof(float), false); d_rv_flags = mem.dev<uint32_t>(reverb_grid_max());
            DevMem tmp(mem.device);  // the f32 IR, only needed to build d_bt
            float* d_ir = tmp.dev<float>((size_t)ich * L, false);
            if (!mem.ok() || !tmp.ok()) return false;
            return FW_CUDA(cudaMemcpy(d_ir, params->ir.data(), (size_t)ich * L * 4, cudaMemcpyHostToDevice)) &&
                   FW_CUDA(launch_reverb_build(d_ir, d_bt, L, ich, nullptr)) && FW_CUDA(cudaDeviceSynchronize());
        }
        if (kind == FW_NODE_RESAMPLER) {
            d_rs_table = mem.dev<float>(params->rs_table.size(), false);
            d_rs_res = mem.dev<uint32_t>(V); d_rs_flags = mem.dev<uint32_t>(V); d_rs_step = mem.dev<uint64_t>(V);
            d_rs_pos = mem.dev<uint64_t>(V);
            if (!mem.ok()) return false;
            if (!FW_CUDA(cudaMemcpy(d_rs_table, params->rs_table.data(), params->rs_table.size() * 4, cudaMemcpyHostToDevice))) return false;
            std::vector<uint64_t> one((size_t)V, 1ull << 32);  // step 1.0 until set; not playing, no resource (zero-initialised)
            return FW_CUDA(cudaMemcpy(d_rs_step, one.data(), (size_t)V * 8, cudaMemcpyHostToDevice));
        }
        if (kind == FW_NODE_SAMPLER) {  // SamplerProcessor::new (sampler.rs:300-320): not playing, playhead 0, no loop, no sample
            d_playing = mem.dev<uint32_t>(V); d_playhead = mem.dev<uint64_t>(V); d_loop_flags = mem.dev<uint32_t>(V);
            d_loop_start = mem.dev<uint64_t>(V); d_loop_end = mem.dev<uint64_t>(V); d_res = mem.dev<uint32_t>(V); d_msg_off = mem.dev<uint32_t>((size_t)V + 1);
            if (!alloc_sampler_staging(std::max<size_t>(4096, 4 * (size_t)V))) return false;
            params->smp_active = true;  // activate() creates the rings (sampler.rs:204-212)
            std::fill(params->smp_pending.begin(), params->smp_pending.end(), (uint16_t)0);
        }
        return true;
    }
    // ---- stream side -------------------------------------------------------------------------------------------------------
    // Sampler messages of one chunk, staged in pinned memory grouped by voice (stable: per-voice order is push order) and copied
    // behind the stream; `ev_staged` says when the copy has left the pinned buffer so that the next chunk may refill it.
    SamplerMsgDev* h_msgs = nullptr; uint32_t* h_off = nullptr; uint32_t* h_cnt = nullptr; cudaEvent_t ev_staged = nullptr; bool staged_pending = false;
    bool alloc_sampler_staging(size_t cap) {
        cap_msgs = cap;
        h_msgs = mem.host<SamplerMsgDev>(cap); h_off = mem.host<uint32_t>((size_t)V + 1); h_cnt = mem.host<uint32_t>((size_t)V + 1);
        d_msgs = mem.dev<SamplerMsgDev>(cap, false);
        return mem.ok() && FW_CUDA(cudaEventCreateWithFlags(&ev_staged, cudaEventDisableTiming));
    }
    // cmds[0..n): the CMD_SAMPLER commands of this node for the chunk, in push order. A chunk without messages leaves d_msg_off all
    // zero: the control kernel reads the offsets of every sampler once any of them has messages.
    bool stage_sampler(const Cmd* const* cmds, uint32_t n, cudaStream_t st) {
        cur_n_msgs = n;
        if (n == 0) {
            if (!msg_off_dirty) return true;
            msg_off_dirty = false;
            return FW_CUDA(cudaMemsetAsync(d_msg_off, 0, ((size_t)V + 1) * sizeof(uint32_t), st));
        }
        if (staged_pending) { cudaEventSynchronize(ev_staged); staged_pending = false; }  // the previous copy has read the pinned buffer (it precedes that chunk's kernels)
        std::memset(h_cnt, 0, ((size_t)V + 1) * sizeof(uint32_t));
        auto each_voice = [&](const Cmd& m, auto&& f) { if (m.voice == FW_ALL_VOICES) { for (uint32_t v = 0; v < V; ++v) f(v); } else if (m.voice < V) f(m.voice); };
        uint64_t total = 0;
        for (uint32_t i = 0; i < n; ++i) each_voice(*cmds[i], [&](uint32_t v) { h_cnt[v + 1]++; ++total; });
        if (total > cap_msgs) { g_dev_err = "sampler message staging overflow"; publish_error(); return false; }
        h_off[0] = 0;
        for (uint32_t v = 0; v < V; ++v) h_off[v + 1] = h_off[v] + h_cnt[v + 1];
        for (uint32_t v = 0; v <= V; ++v) h_cnt[v] = h_off[v];  // running insert positions
        for (uint32_t i = 0; i < n; ++i) { const Cmd& m = *cmds[i]; each_voice(m, [&](uint32_t v) { h_msgs[h_cnt[v]++] = SamplerMsgDev{m.a, m.b, m.x, m.y}; }); }
        cur_n_msgs = (uint32_t)total;
        const bool ok = FW_CUDA(cudaMemcpyAsync(d_msgs, h_msgs, total * sizeof(SamplerMsgDev), cudaMemcpyHostToDevice, st)) &&
                        FW_CUDA(cudaMemcpyAsync(d_msg_off, h_off, ((size_t)V + 1) * sizeof(uint32_t), cudaMemcpyHostToDevice, st));
        cudaEventRecord(ev_staged, st); staged_pending = true; msg_off_dirty = true;
        return ok;
    }
};

struct Plan {
    explicit Plan(int device) : mem(device) {}
    Schedule sched;
    std::vector<std::shared_ptr<NodeDeviceState>> states;   // keeps every referenced node state alive
    std::vector<Id> nodes_to_remove;
    // The control tables: built on the host by lower_control / lower_generic (smp[i].rec / last_play by alloc_plan), laid out as one
    // image and uploaded once by alloc_plan; `tables` then describes the device image.
    std::vector<CtlNode> nodes; std::vector<uint32_t> in_port, out_port; std::vector<SmDesc> sm; std::vector<SamplerCtl> smp; std::vector<RsCtl> rs;
    std::vector<unsigned char> image;  // the tables laid out as CtlTables::image
    CtlTables tables{}; uint64_t* d_flags = nullptr;
    // Data plane: the steps run in order, each one launch group. An operand is C contiguous channels of one space: the caller's input or
    // output rows from channel `index` (row pitch Tfull, or n_in / n_out * Tfull for C == 1), pool buffer `index` of the generic lowering
    // ([buffer][V][chunk], C == 1), or inter-stage scratch d_tmp[index] of the fused chain ([V][C][chunk]).
    enum Space : uint8_t { CALLER_IN, CALLER_OUT, POOL, SCRATCH };
    struct Operand { Space space; uint32_t index, C; };
    struct Step {
        StepKind kind = STEP_PROG;
        // node: the sampler, the biquad or SVF of a temporal step (none: a lone delay), the reverb, resampler or custom node; delay: a
        // temporal step's delay line
        std::shared_ptr<NodeDeviceState> node, delay;
        // PROG launches `prog` once or (`pairs`) per channel pair, an odd last channel narrowed to 1 -> 1. On a master-bus plan the last
        // step is a PROG whose voices run_bus_stage sums into the bus; the generic lowering gives it no output operands.
        ChainProgram prog{}; bool pairs = false;
        int sm0 = -1, sampler_idx = -1, mask_slot = -1, custom_idx = -1;
        std::vector<uint32_t> clear;          // pool buffers cleared before the step: unconnected inputs (schedule.rs:310-313)
        std::vector<Operand> in, out;
    };
    std::vector<Step> steps;
    uint32_t num_buffers = 0;  // generic lowering: pool buffers
    bool reads_caller_rows = false;  // some node reads the caller's input rows directly (row pitch n_in * frames must fit 32 bits)
    std::vector<std::shared_ptr<NodeDeviceState>> samplers;  // index = CtlTables::smp index
    std::shared_ptr<ResTable> res;  // the context's sample resources, which every sampler and resampler reads (null: the plan has neither)
    // c_in / c_out: graph_in's and graph_out's port counts, which the lowerings use; n_in / n_out: the activated stream's channel counts,
    // which lay out the caller's rows. Graph_in ports >= n_in read +0.0, stream inputs >= c_in are ignored, caller output rows >= c_out
    // are written +0.0 and graph_out ports >= n_out are not stored (schedule.rs:213-287, util.rs:96).
    bool bus = false; uint32_t n_sm = 0, c_in = 0, c_out = 0, n_in = 0, n_out = 0, num_voices = 0, block_frames = 0;
    uint32_t bus_width() const { return std::min(c_out, n_out); }  // the master bus's live channels; rows from there on are +0.0
    float* d_zero = nullptr;  // one chunk of +0.0, read with voice stride 0 where the fused chain reads a graph_in port >= n_in
    Records rec{};
    uint64_t* d_bus_mask = nullptr;
    // Per-call scratch, sized on the main thread (lower()) for one chunk of at most `chunk_frames` frames: the stream side
    // never allocates (processor.rs:167-206, context.rs:61-64: the reference's audio thread does not either).
    uint32_t chunk_frames = 0, chunk_blocks = 0;
    bool heavy_stage = false;  // a FIR-reverb GEMM is part of the plan (see run_bus_stage)
    bool graphable = false;  // every by-value kernel argument of a chunk is a function of (buffers, frames): the launch sequence can be replayed as a CUDA graph
    float* d_part[2] = {nullptr, nullptr};     // partial buses [groups][c_out][chunk] and the next radix-16 level
    float* d_tmp[2] = {nullptr, nullptr};      // inter-stage scratch [V][2][chunk]
    float* d_pool = nullptr;                   // generic lowering: [buffer][V][chunk]
    uint16_t* d_slot_of = nullptr;             // sampler graphs: record slot per (block, voice)
    std::vector<uint64_t*> d_custom_masks;     // per custom node (index = Step::custom_idx): dense [block][voice] input masks
    DevMem mem;  // d_flags, the records, d_bus_mask and the scratch; declared last so that it frees them before the node states go
};

// NCCL, resolved at run time with dlopen("libnccl.so.2"): no link-time dependency, and inside a process that
// already loaded torch's bundled NCCL the same copy is reused (same soname). Only the master-bus exchange uses it.
struct NcclUniqueId { char internal[128]; };
struct NcclApi {
    void* handle = nullptr;
    int (*GetUniqueId)(NcclUniqueId*) = nullptr;
    int (*CommInitRank)(void**, int, NcclUniqueId, int) = nullptr;
    int (*AllGather)(const void*, void*, size_t, int, void*, cudaStream_t) = nullptr;
    int (*CommDestroy)(void*) = nullptr;
    const char* (*GetErrorString)(int) = nullptr;
    bool load() {
        if (handle) return true;
        for (const char* name : {"libnccl.so.2", "libnccl.so"}) { handle = dlopen(name, RTLD_NOW | RTLD_GLOBAL); if (handle) break; }
        if (!handle) { g_dev_err = std::string("dlopen(libnccl.so.2) failed: ") + dlerror(); return false; }
        GetUniqueId = reinterpret_cast<decltype(GetUniqueId)>(dlsym(handle, "ncclGetUniqueId"));
        CommInitRank = reinterpret_cast<decltype(CommInitRank)>(dlsym(handle, "ncclCommInitRank"));
        AllGather = reinterpret_cast<decltype(AllGather)>(dlsym(handle, "ncclAllGather"));
        CommDestroy = reinterpret_cast<decltype(CommDestroy)>(dlsym(handle, "ncclCommDestroy"));
        GetErrorString = reinterpret_cast<decltype(GetErrorString)>(dlsym(handle, "ncclGetErrorString"));
        if (!GetUniqueId || !CommInitRank || !AllGather || !CommDestroy || !GetErrorString) { g_dev_err = "libnccl lacks an expected symbol"; return false; }
        return true;
    }
    bool ok(int rc, const char* what) { if (rc == 0) return true; g_dev_err = std::string(what) + ": " + GetErrorString(rc); return false; }
};
static NcclApi g_nccl;

struct CtxToProc { int kind = 0; Plan* plan = nullptr; };                 // 0 NewSchedule, 1 Stop (processor.rs:265-268)
struct ProcToCtx { int kind = 0; Plan* plan = nullptr; void* user_cx = nullptr; };  // 0 ReturnSchedule, 1 Dropped (:270-277)
struct Channels {
    DynSpsc<CtxToProc> to_proc; DynSpsc<ProcToCtx> to_ctx;  // capacity 16 (context.rs:61-64)
    DynSpsc<Cmd> cmds;                        // sampler messages, timed parameter stores, resampler transport (see Cmd); sized from the voice count at activate
    DynSpsc<float*> to_free;                  // CMD_UPLOAD snapshots on their way back to the main thread, which frees them
    std::atomic<uint32_t> drain_epoch{1};     // bumped by the stream side after it emptied `cmds` (per-voice ring-full accounting)
    explicit Channels(size_t cmd_capacity) : to_proc(16), to_ctx(16), cmds(cmd_capacity), to_free(cmd_capacity) {}
    ~Channels() { float* q; while (to_free.pop(&q)) delete[] q; Cmd m; while (cmds.pop(&m)) if (m.kind == CMD_UPLOAD) delete[] reinterpret_cast<float*>(m.x); }
};

}  // namespace fw

using namespace fw;

struct fw_ctx {
    fw_graph_config cfg{};
    std::unique_ptr<Graph> graph;
    std::map<uint64_t, std::shared_ptr<NodeDeviceState>> node_states;  // activated nodes by packed id
    std::string last_error;
    std::shared_ptr<ResTable> res;  // sample resources (created lazily)
    Schedule dbg_schedule; bool dbg_valid = false;
    uint32_t event_block = 0;  // fw_ctx_set_event_block: block offset (into the next call) of the stores and messages that follow
    // ActiveState (context.rs:17-27)
    bool active = false; std::shared_ptr<Channels> ch; uint32_t sample_rate = 0, max_block_frames = 0, n_in = 0, n_out = 0;
    uint32_t max_call_frames = 0;     // longest stretch processed in one go; longer calls are chunked (fw_graph_config::max_call_frames)
    std::unique_ptr<VoiceDetection> voices;  // result of the last successful fw_graph_detect_voices
};

struct fw_processor {
    int device = 0; cudaStream_t stream = nullptr; cudaEvent_t ev[4] = {nullptr, nullptr, nullptr, nullptr};
    std::shared_ptr<Channels> ch; void* user_cx = nullptr;
    Plan* plan = nullptr; bool running = true; bool pending_zero_first = false;
    uint32_t num_voices = 0, max_block_frames = 0, n_in = 0, n_out = 0; bool bus = false;
    float sm_a = 0, sm_b = 0, sm_eps = 0;
    uint64_t launches = 0;
    double cur_stream_time = 0.0; uint32_t cur_stream_status = 0;  // ProcInfo fields of the call being enqueued (node.rs:108-114)
    // I/O staging of the host-buffer entry points, allocated at activate for max_call_frames (the stream side never allocates)
    float *d_in = nullptr, *d_out = nullptr, *d_inter = nullptr, *d_flush = nullptr;
    uint32_t max_call_frames = 0; uint32_t call_epoch = 0, synced_epoch = 0;
    std::vector<Cmd> pend; size_t pend_n = 0; std::vector<const Cmd*> cmd_ptrs;  // drained commands not yet applied (preallocated at activate)
    // CUDA-graph replay of steady chunks (SURVEY f2): the launch sequence of a chunk, captured once per (plan, buffers, frames)
    // res_tab / n_res: the chunk's snapshot of the resource table (see Chunk)
    struct GraphEntry { cudaGraphExec_t exec = nullptr; Plan* plan = nullptr; const float* d_in = nullptr; float* d_out = nullptr; uint32_t t0 = 0, Tc = 0, Tfull = 0;
                        const ResDesc* res_tab = nullptr; uint32_t n_res = 0; uint32_t seen = 0; uint64_t stamp = 0; };
    GraphEntry graphs[4]; uint64_t graph_stamp = 0, graph_replays = 0; bool capturing = false, graphs_off = false;
    // multi-GPU master bus: voices shard by rank; the per-rank buses are all-gathered and tree-summed in rank order
    void* nccl_comm = nullptr; int rank = 0, world = 1;
    float *d_bus_local[2] = {nullptr, nullptr}, *d_gather[2] = {nullptr, nullptr};  // [n_out][chunk], [world][n_out][chunk] per exchange parity: allocated by comm_init
    // the exchange runs on a side stream so that it overlaps the next call's control + chain kernels
    cudaStream_t side = nullptr; cudaEvent_t ev_exchange_done[2] = {nullptr, nullptr}; bool exchange_pending[2] = {false, false};
    uint32_t* d_handover = nullptr; uint32_t xepoch = 0;  // device word main -> side (exchange.cu), exchange counter
    uint64_t* h_masks = nullptr; uint32_t* h_err = nullptr;  // pinned
    // optional per-kernel-class timing (CUDA events on `stream`)
    bool profiling = false; std::vector<cudaEvent_t> prof_ev; std::vector<int> prof_class; size_t prof_used = 0;
    DevMem mem;  // I/O staging, d_flush, the bus exchange buffers, d_handover, h_masks, h_err
    explicit fw_processor(int dev) : device(dev), mem(dev) {}
    // Releases what the handles name; a processor that activate() only partly built has null handles for the rest.
    ~fw_processor() {
        cudaSetDevice(device);
        if (side) cudaStreamDestroy(side);
        for (cudaEvent_t e : ev_exchange_done) if (e) cudaEventDestroy(e);
        if (nccl_comm) g_nccl.CommDestroy(nccl_comm);
        for (cudaEvent_t e : ev) if (e) cudaEventDestroy(e);
        for (cudaEvent_t e : prof_ev) if (e) cudaEventDestroy(e);
        for (auto& g : graphs) if (g.exec) cudaGraphExecDestroy(g.exec);
        if (stream) cudaStreamDestroy(stream);
    }
};

struct ProfScope {  // brackets the launches of one kernel class with a pair of events
    fw_processor* p; bool on;
    ProfScope(fw_processor* p_, int cls) : p(p_), on(false) {
        if (!p->profiling || p->prof_used + 2 > p->prof_ev.size()) return;
        on = true; p->prof_class[p->prof_used / 2] = cls;
        cudaEventRecord(p->prof_ev[p->prof_used], p->stream);
    }
    ~ProfScope() { if (on) { cudaEventRecord(p->prof_ev[p->prof_used + 1], p->stream); p->prof_used += 2; } }
};
// One launch of `n` kernels inside a profile scope of class `cls` (0 control, 1 chain / pointwise, 2 combine, 3 temporal / reverb /
// resampler): false on a CUDA error, else the kernels are counted.
#define FW_LAUNCH(p, cls, n, call) ([&]() -> bool { ProfScope ps_((p), (cls)); if (!FW_CUDA(call)) return false; (p)->launches += (n); return true; }())

// =============================================================================================
// lowering: schedule -> control tables + fused chain program
// =============================================================================================
// The chain op of a node whose kind has one (NodeKind::op.on). sm0: the node's first smoother; its second, if any, is sm0 + 1.
static ChainOp chain_op(const NodeParams& np, int sm0) {
    const NodeKind& nk = node_kind(np.kind);
    ChainOp op{}; op.kind = nk.op.kind; op.sm0 = nk.target[0] ? sm0 : -1; op.sm1 = nk.target[1] ? sm0 + 1 : -1;
    if (nk.op.kind == OP_CLIP) op.f0 = np.threshold_gain;
    return op;
}

// Control tables (one CtlNode per scheduled node, the smoothers, the sampler and resampler transport state) and the node states of
// the plan. sm_of_node[i]: the first smoother of node i, -1: none. Smoothers are numbered in schedule order (the control kernel
// relies on it when it packs their modes).
static bool lower_control(fw_ctx* c, const Schedule& s, Plan* plan, std::vector<int>* sm_of_node, std::string* why) {
    Graph& g = *c->graph;
    const size_t n = s.nodes.size();
    if (n < 2) { *why = "schedule too short for the device control tables"; return false; }
    CtlTables& tb = plan->tables;
    tb.n_nodes = (uint32_t)n; tb.n_buffers = s.num_buffers; tb.n_flag_words = std::max(1u, (s.num_buffers + 63u) / 64u);
    if (control_threads(tb.n_flag_words, c->cfg.device) == 0) { *why = "the silence flags of one voice do not fit in the device's shared memory"; return false; }
    uint32_t n_sm = 0;
    sm_of_node->assign(n, -1);
    plan->nodes.assign(n, CtlNode{});
    for (size_t i = 0; i < n; ++i) {
        const SchedNode& sn = s.nodes[i];
        NodeRec* nr = g.node(sn.id);
        CtlNode& cn = plan->nodes[i];
        cn.kind = (uint8_t)nr->params->kind; cn.n_in = (uint8_t)sn.in.size(); cn.n_out = (uint8_t)sn.out.size();
        cn.in_off = (uint32_t)plan->in_port.size(); cn.out_off = (uint32_t)plan->out_port.size(); cn.sm0 = cn.sm1 = -1;
        if (nr->params->kind == FW_NODE_CUSTOM) cn.sm0 = (int32_t)nr->params->custom->info.out_silence_rule;
        for (const InAssign& a : sn.in) plan->in_port.push_back(a.buffer | (a.should_clear ? kPortClear : 0u));
        for (const OutAssign& a : sn.out) plan->out_port.push_back(a.buffer);
        auto it = c->node_states.find(sn.id.pack());
        if (it == c->node_states.end()) { *why = "internal: node without device state"; return false; }
        std::shared_ptr<NodeDeviceState> st = it->second;
        plan->states.push_back(st);
        if (st->n_sm) {
            (*sm_of_node)[i] = (int)n_sm;
            cn.sm0 = (int32_t)n_sm; if (st->n_sm == 2) cn.sm1 = (int32_t)(n_sm + 1);
            for (uint32_t k = 0; k < st->n_sm; ++k, ++n_sm) plan->sm.push_back(SmDesc{st->sm_input[k], st->sm_last[k], st->sm_status[k], st->d_target[k]});
        }
    }
    tb.n_smoothers = n_sm; plan->n_sm = n_sm;
    for (size_t i = 0; i < n; ++i) {  // SamplerNodes: per-voice transport state lives in the node's device state
        if (plan->nodes[i].kind != FW_NODE_SAMPLER) continue;
        const std::shared_ptr<NodeDeviceState>& st = plan->states[i];
        SamplerCtl sc{};
        sc.playing = st->d_playing; sc.playhead = st->d_playhead; sc.loop_flags = st->d_loop_flags; sc.loop_start = st->d_loop_start; sc.loop_end = st->d_loop_end; sc.res = st->d_res;
        sc.msgs = st->d_msgs; sc.msg_off = st->d_msg_off;
        sc.n_out = (uint32_t)s.nodes[i].out.size();
        plan->nodes[i].sm1 = (int32_t)plan->smp.size();
        plan->smp.push_back(sc);
        plan->samplers.push_back(st);
    }
    for (size_t i = 0; i < n; ++i) {
        if (plan->nodes[i].kind != FW_NODE_RESAMPLER) continue;
        const std::shared_ptr<NodeDeviceState>& st = plan->states[i];
        plan->nodes[i].sm1 = (int32_t)plan->rs.size();
        plan->rs.push_back(RsCtl{st->d_rs_flags, st->d_rs_res, (uint32_t)s.nodes[i].out.size(), 0u});
    }
    tb.n_samplers = (uint32_t)plan->smp.size(); tb.n_resamplers = (uint32_t)plan->rs.size();
    if (tb.n_samplers || tb.n_resamplers) plan->res = c->res;
    tb.n_in_ports = (uint32_t)plan->in_port.size(); tb.n_out_ports = (uint32_t)plan->out_port.size();
    return true;
}

// Appends `op` to a chain program and gives its smoothers program-local indices (ChainOp::l0 / l1, ChainProgram::sm). False, and the
// program unchanged, when the program would read more than kMaxProgSmoothers distinct smoothers.
static bool prog_push(ChainProgram& p, ChainOp op) {
    uint32_t n_sm = p.n_sm;
    int32_t sm[kMaxProgSmoothers];
    std::copy(p.sm, p.sm + kMaxProgSmoothers, sm);
    const int32_t g[2] = {op.sm0, op.sm1};
    int32_t* l[2] = {&op.l0, &op.l1};
    for (int k = 0; k < 2; ++k) {
        *l[k] = -1;
        if (g[k] < 0) continue;
        uint32_t i = 0;
        while (i < n_sm && sm[i] != g[k]) ++i;
        if (i == n_sm) { if (n_sm == (uint32_t)kMaxProgSmoothers) return false; sm[n_sm++] = g[k]; }
        *l[k] = (int32_t)i;
    }
    std::copy(sm, sm + kMaxProgSmoothers, p.sm); p.n_sm = n_sm;
    p.ops[p.n_ops++] = op;
    return true;
}

// Data plane, first choice: a linear chain graph_in -> n1 -> ... -> nk -> graph_out, port i to port i, fused into stages. Stage 0
// reads the caller's rows, stage si writes scratch si & 1 and the last stage the caller's output rows. False, with the reason, for
// any other schedule.
static bool lower_chain(const Schedule& s, const std::vector<int>& sm_of_node, bool bus, Plan* plan, std::string* why) {
    const size_t n = s.nodes.size();
    const SchedNode& gin = s.nodes.front();
    const SchedNode& gout = s.nodes.back();
    std::vector<Plan::Step>& steps = plan->steps;
    uint32_t width = (uint32_t)gin.out.size();
    // a stage of `width` channels in and out (the space and index of its operands are set at the end)
    auto stage = [&](StepKind kind, const std::shared_ptr<NodeDeviceState>& node) {
        Plan::Step sp; sp.kind = kind; sp.node = node;
        sp.in = {Plan::Operand{Plan::SCRATCH, 0, width}}; sp.out = sp.in;
        steps.push_back(std::move(sp));
    };
    Id prev = gin.id;
    size_t first = 1;
    if (width == 0 && n >= 3 && plan->nodes[1].kind == FW_NODE_SAMPLER && s.nodes[1].in.empty() && s.nodes[1].out.size() >= 1 && s.nodes[1].out.size() <= 2) {
        // no stream inputs: a SamplerNode heads the chain (BASELINE config 5: sampler -> gain -> pan -> ... -> bus)
        width = (uint32_t)s.nodes[1].out.size();
        stage(STEP_SAMPLER, plan->states[1]);
        steps.back().in.clear(); steps.back().sm0 = sm_of_node[1]; steps.back().sampler_idx = plan->nodes[1].sm1;
        prev = s.nodes[1].id; first = 2;
    }
    if (width < 1 || width > 2) { *why = "the fused chain supports 1 or 2 channels"; return false; }
    const uint32_t head_width = first == 1 ? width : 0u;  // graph_in ports the first stage reads from the caller's rows
    auto fed_by_prev = [&](const SchedNode& sn, uint32_t w) {
        if (sn.in.size() != w) return false;
        for (uint32_t p = 0; p < w; ++p) if (sn.in[p].should_clear || sn.in[p].producer != prev || sn.in[p].producer_port != p) return false;
        return true;
    };
    ChainProgram cur{}; cur.c_in = width;  // the pointwise stage being accumulated
    auto close_pointwise = [&](bool force) {
        if (cur.n_ops > 0 || force) { cur.c_out = width; stage(STEP_PROG, nullptr); steps.back().prog = cur; steps.back().in[0].C = cur.c_in; }
        cur = ChainProgram{}; cur.c_in = width;
    };
    for (size_t i = first; i + 1 < n; ++i) {
        const SchedNode& sn = s.nodes[i];
        const NodeParams& np = *plan->states[i]->params;
        if (!fed_by_prev(sn, width)) { *why = "voice graph is not a linear port-to-port chain"; return false; }
        if (sn.out.size() < 1 || sn.out.size() > 2) { *why = "the fused chain supports 1 or 2 channels"; return false; }
        const uint32_t kind = np.kind;
        const NodeKind& nk = node_kind(kind);
        if (nk.step == STEP_TEMPORAL || nk.step == STEP_REVERB) {
            const std::shared_ptr<NodeDeviceState>& st = plan->states[i];
            // a delay directly after a biquad joins its pass; anything else opens a new stage
            if (kind == FW_NODE_DELAY && !steps.empty() && steps.back().kind == STEP_TEMPORAL && !steps.back().delay &&
                steps.back().node && steps.back().node->kind == FW_NODE_BIQUAD && cur.n_ops == 0) {
                steps.back().delay = st;
            } else {
                close_pointwise(false);
                stage(nk.step, kind == FW_NODE_DELAY ? nullptr : st);
                if (kind == FW_NODE_DELAY) steps.back().delay = st;
            }
            prev = sn.id;
            continue;
        }
        if (cur.n_ops >= (uint32_t)kMaxChainOps) { *why = "more than 16 pointwise nodes in a row"; return false; }
        if (kind == FW_NODE_SUM) {
            if (sn.in.size() == sn.out.size()) { prev = sn.id; continue; }  // 1-port sum == copy (sum.rs:58-65): no data op
            *why = "SumNode with more than one port inside a voice chain"; return false;
        }
        if (!nk.op.on) { *why = std::string("node kind '") + nk.name + "' has no device lowering yet"; return false; }
        const ChainOp op = chain_op(np, sm_of_node[i]);
        if (!prog_push(cur, op)) { close_pointwise(false); prog_push(cur, op); }  // a program reads at most kMaxProgSmoothers smoothers
        width = (uint32_t)sn.out.size();
        prev = sn.id;
    }
    if (!fed_by_prev(gout, width)) { *why = "graph_out is not fed port-to-port by the end of the chain"; return false; }
    // the last stage must be pointwise when the master bus follows it, and a plan is never empty
    close_pointwise(steps.empty() || (bus && cur.n_ops == 0 && steps.back().kind != STEP_PROG));
    // Only a pointwise stage addresses the caller's rows channel by channel (a voice stride of n_in / n_out rows, zero rows for graph_in
    // ports >= n_in, graph_out ports >= n_out left out); a temporal or sampler stage reads and writes [V][C] rows.
    if ((head_width && head_width != plan->n_in && steps.front().kind != STEP_PROG) ||
        (!bus && width != plan->n_out && steps.back().kind != STEP_PROG)) {
        *why = "a stateful stage at the end of the chain on a stream whose channel counts differ from the graph's ports"; return false;
    }
    for (uint32_t si = 0; si < steps.size(); ++si) {
        const bool last = si + 1 == steps.size();
        for (Plan::Operand& o : steps[si].in) o = si == 0 ? Plan::Operand{Plan::CALLER_IN, 0, o.C} : Plan::Operand{Plan::SCRATCH, (si - 1) & 1, o.C};
        for (Plan::Operand& o : steps[si].out) o = last ? Plan::Operand{Plan::CALLER_OUT, 0, o.C} : Plan::Operand{Plan::SCRATCH, si & 1, o.C};
    }
    plan->c_out = width;
    return true;
}

static_assert(kMaxBusChannels == FW_MAX_BUS_CHANNELS, "plan.hpp and the C header name the same bus limit");

// Data plane, general case: the reference's own buffer assignment on device, one step per scheduled node over pool buffers. graph_in
// copies the caller's rows to the pool, graph_out the pool to the caller's rows or the bus (prepare_graph_inputs / read_graph_outputs,
// schedule.rs:213-287).
static bool lower_generic(const Schedule& s, const std::vector<int>& sm_of_node, bool bus, Plan* plan, std::string* why) {
    const size_t n = s.nodes.size();
    plan->steps.clear(); plan->num_buffers = s.num_buffers;
    if (bus && plan->bus_width() > (uint32_t)kMaxBusChannels) { *why = "master bus over more than 8 graph_out channels (FW_MAX_BUS_CHANNELS)"; return false; }
    uint32_t n_mask_slots = 0;  // nodes whose data-plane body needs the per-block input silence mask
    for (size_t i = 0; i < n; ++i) {
        const SchedNode& sn = s.nodes[i];
        const NodeParams& np = *plan->states[i]->params;
        const uint32_t kind = np.kind;
        const bool endpoint = i == 0 || i + 1 == n;
        Plan::Step sp; sp.node = plan->states[i]; sp.sm0 = sm_of_node[i];
        for (const InAssign& a : sn.in) { sp.in.push_back(Plan::Operand{Plan::POOL, a.buffer, 1}); if (a.should_clear) sp.clear.push_back(a.buffer); }
        for (const OutAssign& a : sn.out) sp.out.push_back(Plan::Operand{Plan::POOL, a.buffer, 1});
        // graph_in copies the stream's channels and clears its ports >= n_in; graph_out stores its ports < n_out (schedule.rs:244-252,269)
        if (i == 0) for (uint32_t p = 0; p < sn.out.size(); ++p) {
            if (p < plan->n_in) sp.in.push_back(Plan::Operand{Plan::CALLER_IN, p, 1}); else sp.clear.push_back(sn.out[p].buffer);
        }
        if (i + 1 == n && !bus) for (uint32_t p = 0; p < sn.in.size() && p < plan->n_out; ++p) sp.out.push_back(Plan::Operand{Plan::CALLER_OUT, p, 1});
        const NodeKind& nk = node_kind(kind);
        sp.kind = kind == FW_NODE_SUM && sn.in.size() == sn.out.size() ? STEP_PROG : nk.step;  // a 1-port SumNode is a copy (sum.rs:58-65)
        // bodies that branch on the input silence mask (see silence_fix_kernel / sum_kernel)
        const bool needs_mask = !endpoint && (sp.kind == STEP_CUSTOM || (!sn.out.empty() && (sp.kind == STEP_SUM || (nk.op.mask && !(kind == FW_NODE_VOLUME && sn.in.size() == 2)))));
        if (kind == FW_NODE_CUSTOM && !np.custom->vt.process_device) { *why = std::string("custom node '") + np.custom->debug_name + "' has no process_device: it cannot run on the device (there is no CPU fallback)"; return false; }
        if (needs_mask) {
            sp.mask_slot = (int)n_mask_slots; plan->nodes[i].mask_slot = ++n_mask_slots;
        }
        if (kind == FW_NODE_DUMMY && !endpoint && !sn.out.empty()) { *why = "a DummyAudioNode inside the graph leaves its outputs stale in the reference (dummy.rs:34-41): not reproducible on the device"; return false; }
        if (kind == FW_NODE_MONO_TO_STEREO && (sn.in.size() != 1 || sn.out.size() != 2)) { *why = "MonoToStereoNode must be 1 -> 2"; return false; }
        if (kind == FW_NODE_STEREO_TO_MONO && (sn.in.size() != 2 || sn.out.size() != 1)) { *why = "StereoToMonoNode must be 2 -> 1"; return false; }
        // The program: the node's op, else a copy for graph_in, graph_out (both Dummy nodes), a 1-port SumNode and a Dummy node inside the
        // graph, which has no outputs and so launches nothing. It runs per channel pair where the body works channel by channel, else once
        // for the node; fuse_generic makes a stereo Volume it fuses, or that reads the caller's rows, one launch too. With a master bus, the
        // bus stage takes graph_out's channels at once.
        if (nk.op.on) {
            prog_push(sp.prog, chain_op(np, sp.sm0));
            sp.prog.c_in = nk.op.c_in; sp.prog.c_out = nk.op.c_out; sp.pairs = nk.op.pairs;
        } else if (sp.kind == STEP_PROG) {
            const bool bus_out = bus && i + 1 == n;
            sp.prog.c_in = sp.prog.c_out = bus_out ? (uint32_t)sn.in.size() : 2u; sp.pairs = !bus_out;
        }
        if (kind == FW_NODE_DELAY) std::swap(sp.node, sp.delay);
        if (kind == FW_NODE_SAMPLER) sp.sampler_idx = plan->nodes[i].sm1;
        plan->steps.push_back(std::move(sp));
    }
    plan->rec.n_mask_slots = n_mask_slots;
    return true;
}

// Generic lowering, second step (SURVEY f2: "fuse runs of pointwise nodes between fan-out points"):
//  * a run of mask-independent pointwise nodes (stereo Volume, Pan) that are adjacent in the schedule and feed each other port to
//    port with no other consumer becomes one chain program, launched where its last node stands; graph_out (copy to the caller's
//    rows, or the bus stage) can be that last node. Adjacency makes the fused launch read and write its pool buffers at the same
//    point of the schedule as the unfused nodes did, so the compiler's buffer reuse (compiler.rs:302-412) stays valid; a run whose
//    last outputs reuse the buffers of its first inputs is not fused (no in-place launches).
//  * a run head or a Biquad / SVF / Delay node fed entirely by graph_in reads the caller's input rows itself (pointer + pitch),
//    first-block zeroing after a schedule swap (Q11) included; if every consumer of graph_in does, the pool copy of the inputs is skipped.
static void fuse_generic(const Schedule& s, Plan* plan) {
    const size_t n = s.nodes.size();
    std::vector<Plan::Step>& st = plan->steps;  // one per scheduled node until the end
    auto nk = [&](size_t i) -> const NodeKind& { return node_kind(plan->states[i]->kind); };
    std::unordered_map<uint64_t, size_t> index_of;
    for (size_t i = 0; i < n; ++i) index_of[s.nodes[i].id.pack()] = i;
    std::vector<std::vector<uint32_t>> n_cons(n);
    for (size_t i = 0; i < n; ++i) n_cons[i].assign(s.nodes[i].out.size(), 0u);
    for (size_t i = 0; i < n; ++i) for (const InAssign& a : s.nodes[i].in) {
        if (a.should_clear) continue;
        auto it = index_of.find(a.producer.pack());
        if (it != index_of.end() && a.producer_port < n_cons[it->second].size()) n_cons[it->second][a.producer_port]++;
    }
    auto connected = [&](size_t i) { for (const InAssign& a : s.nodes[i].in) if (a.should_clear) return false; return true; };
    auto stereo_pointwise = [&](size_t i) {
        return i > 0 && i + 1 < n && nk(i).op.fuses && s.nodes[i].in.size() == 2 && s.nodes[i].out.size() == 2 &&
               st[i].mask_slot < 0 && connected(i);
    };
    auto fed_only_by = [&](size_t i, size_t j) {  // node i's inputs are node j's outputs, port to port, and nothing else reads them
        if (s.nodes[i].in.size() != s.nodes[j].out.size()) return false;
        for (size_t p = 0; p < s.nodes[i].in.size(); ++p) {
            const InAssign& a = s.nodes[i].in[p];
            if (a.should_clear || a.producer != s.nodes[j].id || a.producer_port != p || n_cons[j][p] != 1) return false;
        }
        return true;
    };
    std::vector<bool> folded(n, false);  // runs inside the step that ends its run; graph_in: every reader reads the caller's rows
    // graph_in aliasing: which nodes can read the caller's rows, and is the pool copy still needed
    std::vector<uint32_t> alias_cons(s.nodes[0].out.size(), 0u);
    for (size_t i = 1; i + 1 < n; ++i) {
        if (!(stereo_pointwise(i) || (nk(i).step == STEP_TEMPORAL && connected(i) && !s.nodes[i].in.empty()))) continue;
        bool all = true;
        for (const InAssign& a : s.nodes[i].in) if (a.producer != s.nodes[0].id || a.producer_port >= alias_cons.size() || a.producer_port >= plan->n_in) all = false;
        if (!all) continue;
        for (size_t k = 0; k < s.nodes[i].in.size(); ++k) {
            const uint32_t port = s.nodes[i].in[k].producer_port;
            st[i].in[k] = Plan::Operand{Plan::CALLER_IN, port, 1};
            alias_cons[port]++;
        }
        st[i].pairs = false;
        plan->reads_caller_rows = true;
    }
    folded[0] = true;
    for (size_t p = 0; p < alias_cons.size(); ++p) if (n_cons[0][p] > alias_cons[p]) folded[0] = false;
    // runs: node i extends the run that ends at node j = i - 1 by its own op (graph_out adds none)
    for (size_t i = 2; i < n; ++i) {
        const size_t j = i - 1;
        const bool tail = i + 1 == n && s.nodes[i].in.size() == 2;
        if (!(stereo_pointwise(i) || tail) || !stereo_pointwise(j) || !fed_only_by(i, j)) continue;
        if (st[j].prog.n_ops + 1 > (uint32_t)kMaxChainOps) continue;
        bool in_place = false;
        for (const Plan::Operand& o : st[i].out) for (const Plan::Operand& q : st[j].in) if (o.space == q.space && o.index == q.index) in_place = true;
        if (in_place) continue;
        ChainProgram pr = st[j].prog;
        bool fits = true;  // the run closes before its program would read more than kMaxProgSmoothers smoothers
        for (uint32_t k = 0; k < st[i].prog.n_ops && fits; ++k) fits = prog_push(pr, st[i].prog.ops[k]);
        if (!fits) continue;
        st[i].prog = pr; st[i].pairs = false;
        st[i].in = st[j].in;
        folded[j] = true;
    }
    std::vector<Plan::Step> kept;
    for (size_t i = 0; i < n; ++i) if (!folded[i]) kept.push_back(std::move(st[i]));
    st = std::move(kept);
}

// Device buffers of the plan (main thread): the record buffers, the silence flags and the per-call scratch of one chunk.
static bool alloc_plan(const fw_ctx* c, Plan* plan, bool pool, std::string* why) {
    const uint32_t V = c->cfg.num_voices, F = c->max_block_frames, n_sm = plan->n_sm;
    plan->num_voices = V; plan->block_frames = F; plan->bus = c->cfg.master_bus != 0;
    DevMem& mem = plan->mem;
    plan->d_flags = mem.dev<uint64_t>((size_t)plan->tables.n_flag_words * V);
    Records& r = plan->rec;
    r.n_smoothers = n_sm; r.n_mode_words = std::max(1u, (n_sm + kModesPerWord - 1) / kModesPerWord);
    // Longest transient a record buffer must hold: a ramp decays like b^n with tau = smooth_secs * sample_rate samples and settles at
    // |delta| * b^n < 1e-5 (smoother.rs:99-100,179); sized for |delta| up to 1e4 (a jump of 10000 % in percent_volume): ln(1e9) tau.
    // A chunk never has more blocks than chunk_blocks, so min() with that is enough when the chunk is shorter than the ramp.
    {
        const double tau = 0.01 * (double)c->sample_rate;
        const uint32_t ramp_blocks = (uint32_t)std::ceil(20.8 * tau / (double)F) + 4u;
        const uint32_t kc = (c->max_call_frames + F - 1) / F + 1u;
        r.kt_max = (n_sm ? ramp_blocks : 4u) + 8u * (uint32_t)plan->samplers.size();  // every sample that ends mid-call opens a short transient of its own
        r.kt_max = std::max(2u, std::min(r.kt_max, kc));
    }
    r.modes = mem.dev<uint32_t>(r.modes_count(V));
    r.vals = mem.dev<float>(r.vals_count(V));
    r.curves = mem.dev<float>(r.curves_count(V, F), false);
    r.steady_k = mem.dev<uint32_t>(V);
    r.gout_mask = mem.dev<uint64_t>(V);
    r.st_modes = mem.dev<uint32_t>(V);
    r.st_vals = mem.dev<float>(r.st_vals_count(V));
    r.in_masks = mem.dev<uint64_t>(r.in_masks_count(V));
    r.st_in_masks = mem.dev<uint64_t>(r.st_in_masks_count(V));
    r.error = mem.dev<uint32_t>(1);
    plan->d_bus_mask = mem.dev<uint64_t>(1);
    {   // per-call scratch for one chunk (see Plan)
        const uint32_t Tc = c->max_call_frames, Kc = (Tc + F - 1) / F;
        plan->chunk_frames = Tc; plan->chunk_blocks = Kc;
        const uint32_t n_out = plan->bus_width(), groups = chain_voice_groups(V);
        if (plan->bus) {
            plan->d_part[0] = mem.dev<float>((size_t)groups * n_out * Tc, false); plan->d_part[1] = mem.dev<float>((size_t)((groups + 15) / 16) * n_out * Tc, false);
        }
        for (const Plan::Step& sp : plan->steps)
            for (const Plan::Operand& o : sp.out) if (o.space == Plan::SCRATCH && !plan->d_tmp[o.index]) plan->d_tmp[o.index] = mem.dev<float>((size_t)V * 2 * Tc, false);
        if (pool) plan->d_pool = mem.dev<float>((size_t)plan->num_buffers * V * Tc, false);
        else if (plan->n_in < plan->c_in) plan->d_zero = mem.dev<float>(Tc);
        if (!plan->samplers.empty()) {
            plan->d_slot_of = mem.dev<uint16_t>(Records::kv_count(Kc, V));
            for (size_t i = 0; i < plan->samplers.size(); ++i) {
                plan->smp[i].rec = mem.dev<SmpRec>(Records::kv_count(Kc, V)); plan->smp[i].last_play = mem.dev<uint32_t>(V);
            }
        }
        for (auto& sp : plan->steps) if (sp.kind == STEP_CUSTOM) { sp.custom_idx = (int)plan->d_custom_masks.size(); plan->d_custom_masks.push_back(mem.dev<uint64_t>(Records::kv_count(Kc, V))); }
        r.slot_of = plan->d_slot_of;
    }
    {   // the control tables as one image (CtlTables), uploaded once
        CtlTables& tb = plan->tables;
        std::vector<unsigned char>& im = plan->image;
        auto put = [&](const auto& h) {
            const size_t o = im.size(), n = h.size() * sizeof(h[0]);
            im.resize(o + ((n + 15) & ~(size_t)15));
            if (n) std::memcpy(im.data() + o, h.data(), n);
            return o;
        };
        const size_t o_nodes = put(plan->nodes), o_in = put(plan->in_port), o_out = put(plan->out_port), o_sm = put(plan->sm), o_smp = put(plan->smp), o_rs = put(plan->rs);
        unsigned char* d = mem.dev<unsigned char>(im.size(), false);
        if (!d || (!im.empty() && !FW_CUDA(cudaMemcpy(d, im.data(), im.size(), cudaMemcpyHostToDevice)))) { *why = "control table upload failed: " + g_dev_err; return false; }
        tb.image = d; tb.image_bytes = (uint32_t)im.size();
        tb.o_nodes = (uint32_t)o_nodes; tb.o_in_port = (uint32_t)o_in; tb.o_out_port = (uint32_t)o_out; tb.o_sm = (uint32_t)o_sm; tb.o_smp = (uint32_t)o_smp; tb.o_rs = (uint32_t)o_rs;
    }
    if (!mem.ok()) { *why = "device allocation failed: " + g_dev_err; return false; }
    return true;
}

static bool lower(fw_ctx* c, const Schedule& s, Plan* plan, std::string* why) {
    std::vector<int> sm_of_node;
    if (!lower_control(c, s, plan, &sm_of_node, why)) return false;
    const SchedNode& gin = s.nodes.front();
    const SchedNode& gout = s.nodes.back();
    plan->c_in = (uint32_t)gin.out.size(); plan->c_out = (uint32_t)gout.in.size(); plan->n_in = c->n_in; plan->n_out = c->n_out;
    const bool bus = c->cfg.master_bus != 0;
    const bool chain = lower_chain(s, sm_of_node, bus, plan, why);
    if (!chain) {
        if (!lower_generic(s, sm_of_node, bus, plan, why)) return false;
        fuse_generic(s, plan);
    }
    if (!alloc_plan(c, plan, !chain, why)) return false;
    plan->graphable = true;
    for (auto& st : plan->states) if (node_kind(st->kind).call_varying) plan->graphable = false;
    for (auto& st : plan->states) if (st->kind == FW_NODE_CONV_REVERB) plan->heavy_stage = true;
    return true;
}

static std::shared_ptr<NodeParams> params_from_desc(const fw_node_desc* d, uint32_t V) {
    auto p = std::make_shared<NodeParams>();
    p->kind = d->kind; p->num_voices = V;
    switch (d->kind) {
        case FW_NODE_DUMMY: case FW_NODE_SUM: case FW_NODE_MONO_TO_STEREO: case FW_NODE_STEREO_TO_MONO: break;
        case FW_NODE_VOLUME: {  // volume.rs:16-24
            float pct = std::fmax(d->f0, 0.0f), n = std::fmax(pct, 0.0f) * (1.0f / 100.0f);
            p->percent.assign(V, pct); p->raw_gain.assign(V, n * n);
            break;
        }
        case FW_NODE_SAMPLER: {  // sampler.rs:56-66
            float pct = std::fmax(d->f0, 0.0f), n = std::fmax(pct, 0.0f) * (1.0f / 100.0f);
            p->percent.assign(V, pct); p->raw_gain.assign(V, n * n);
            p->smp_playing.assign(V, 0); p->smp_pending.assign(V, 0); p->smp_pending_epoch.assign(V, 0);
            break;
        }
        case FW_NODE_HARD_CLIP:  // hard_clip.rs:8-12, util.rs:21-27
            p->threshold_gain = d->f0 <= -100.0f ? 0.0f : std::pow(10.0f, 0.05f * d->f0);
            break;
        case FW_NODE_PAN: {
            double pp = std::fmin(std::fmax((double)d->f0, -1.0), 1.0), th = (pp + 1.0) * (M_PI / 4.0);
            p->pan.assign(V, d->f0); p->gain_l.assign(V, (float)std::cos(th)); p->gain_r.assign(V, (float)std::sin(th));
            break;
        }
        case FW_NODE_BIQUAD: case FW_NODE_SVF: {  // identity stages: biquad b0 = 1; SVF a1 = m0 = 1
            const uint32_t w = coeff_width(d->kind);
            p->num_stages = d->u0 > 8 ? 8 : d->u0;
            p->coeffs.assign((size_t)V * p->num_stages * w, 0.0f);
            for (size_t i = 0; i < (size_t)V * p->num_stages; ++i) { p->coeffs[i * w] = 1.0f; if (d->kind == FW_NODE_SVF) p->coeffs[i * w + 3] = 1.0f; }
            break;
        }
        case FW_NODE_DELAY: p->delay = d->u0; break;
        case FW_NODE_RESAMPLER:
            if (!d->data || d->u0 == 0 || d->u1 == 0 || d->data_len < (uint64_t)d->u0 * d->u1) return nullptr;
            p->rs_phases = d->u0; p->rs_taps = d->u1; p->rs_table.assign(d->data, d->data + (size_t)d->u0 * d->u1);
            break;
        case FW_NODE_CONV_REVERB:
            if (!d->data || d->data_len < (uint64_t)d->u0 * d->u1) return nullptr;
            p->ir_len = d->u0; p->ir_channels = d->u1; p->ir.assign(d->data, d->data + (size_t)d->u0 * d->u1);
            break;
        default: return nullptr;
    }
    return p;
}

static void ctx_drain(fw_ctx* c, bool* dropped, void** cx) {  // context.rs:213-234
    if (!c->active) return;
    ProcToCtx m;
    while (c->ch->to_ctx.pop(&m)) {
        if (m.kind == 0) { delete m.plan; }  // on_schedule_returned: removed processors are released here, on the main thread
        else { delete m.plan; *dropped = true; *cx = m.user_cx; }
    }
}
static void ctx_graph_deactivate(fw_ctx* c) {  // graph.rs:671-689
    c->node_states.clear();
    c->graph->nodes_removed_since_compile.clear();
    c->graph->mark_dirty();
    c->graph->nodes_to_activate.clear();
    c->graph->each_node([&](Id id, NodeRec& r) { r.activated = false; c->graph->nodes_to_activate.push_back(id); });
}

extern "C" {

void fw_graph_config_default(fw_graph_config* c) { *c = fw_graph_config{0, 2, 64, 256, 1, 0, 0, 0}; }

fw_ctx* fw_ctx_new(const fw_graph_config* cfg) {
    if (!cfg || cfg->num_voices == 0 || cfg->num_graph_inputs > 64 || cfg->num_graph_outputs > 64) { g_dev_err = "bad graph config"; return nullptr; }
    auto* c = new fw_ctx();
    c->cfg = *cfg;
    c->graph = std::make_unique<Graph>(cfg->num_graph_inputs, cfg->num_graph_outputs, cfg->num_voices);
    return c;
}
void fw_ctx_free(fw_ctx* c) {
    if (!c) return;
    if (c->active) {  // Drop for FirewheelGraphCtx (context.rs:236-242): deactivate, then release what is still queued either way
        fw_ctx_deactivate(c, 1);
    }
    c->node_states.clear();
    delete c;
}
const char* fw_ctx_last_error(fw_ctx* c) { return c ? c->last_error.c_str() : "null context"; }
fw_node_id fw_graph_in_node(fw_ctx* c) { return c->graph->graph_in().pack(); }
fw_node_id fw_graph_out_node(fw_ctx* c) { return c->graph->graph_out().pack(); }

fw_node_id fw_graph_add_node(fw_ctx* c, uint32_t ni, uint32_t no, const fw_node_desc* d) {
    if (!c || !d || ni > 64 || no > 64) return FW_ID_DANGLING;
    auto p = params_from_desc(d, c->cfg.num_voices);
    if (!p) { c->last_error = "bad node description"; return FW_ID_DANGLING; }
    return c->graph->add_node(ni, no, std::move(p)).pack();
}
fw_node_id fw_graph_add_custom_node(fw_ctx* c, uint32_t ni, uint32_t no, const fw_node_vtable* vt, void* node) {  // graph.rs:201-231
    if (!c || !vt || ni > 64 || no > 64 || !vt->debug_name || !vt->info || !vt->activate) {
        if (vt && vt->drop_node) vt->drop_node(node);
        if (c) c->last_error = "bad custom node (vtable needs debug_name, info and activate)";
        return FW_ID_DANGLING;
    }
    auto p = std::make_shared<NodeParams>();
    p->kind = FW_NODE_CUSTOM; p->num_voices = c->cfg.num_voices;
    p->custom = std::make_shared<CustomNode>();
    p->custom->vt = *vt; p->custom->node = node;
    const char* name = vt->debug_name(node);
    p->custom->debug_name = name ? name : "custom";
    vt->info(node, &p->custom->info);  // `let info = node.info()` (graph.rs:210)
    return c->graph->add_node(ni, no, std::move(p)).pack();
}
static void write_ids(const std::vector<Id>& v, uint64_t* out, uint32_t cap, uint32_t* n) {
    if (n) *n = (uint32_t)v.size();
    for (size_t i = 0; i < v.size() && i < cap && out; ++i) out[i] = v[i].pack();
}
int fw_graph_remove_node(fw_ctx* c, fw_node_id node, fw_edge_id* removed, uint32_t cap, uint32_t* n_removed) {
    std::vector<Id> rm;
    if (!c->graph->remove_node(Id::unpack(node), &rm)) { if (n_removed) *n_removed = 0; return -1; }
    write_ids(rm, removed, cap, n_removed);
    return 0;
}
int fw_graph_set_num_inputs(fw_ctx* c, fw_node_id node, uint32_t n, fw_edge_id* removed, uint32_t cap, uint32_t* n_removed) {
    std::vector<Id> rm;
    if (n > 64 || !c->graph->set_num_inputs(Id::unpack(node), n, &rm)) { if (n_removed) *n_removed = 0; return -1; }
    write_ids(rm, removed, cap, n_removed);
    return 0;
}
int fw_graph_set_num_outputs(fw_ctx* c, fw_node_id node, uint32_t n, fw_edge_id* removed, uint32_t cap, uint32_t* n_removed) {
    std::vector<Id> rm;
    if (n > 64 || !c->graph->set_num_outputs(Id::unpack(node), n, &rm)) { if (n_removed) *n_removed = 0; return -1; }
    write_ids(rm, removed, cap, n_removed);
    return 0;
}
int fw_graph_connect(fw_ctx* c, fw_node_id src, uint32_t sp, fw_node_id dst, uint32_t dp, int check, fw_edge_id* out_edge, fw_node_id* err_node, uint32_t* err_port) {
    Id e;
    int rc = c->graph->connect(Id::unpack(src), sp, Id::unpack(dst), dp, check != 0, &e);
    if (rc == FW_EDGE_OK) { if (out_edge) *out_edge = e.pack(); return rc; }
    if (err_node) {
        switch (rc) {
            case FW_EDGE_SRC_NODE_NOT_FOUND: case FW_EDGE_OUT_PORT_OUT_OF_RANGE: *err_node = src; break;
            case FW_EDGE_DST_NODE_NOT_FOUND: case FW_EDGE_IN_PORT_OUT_OF_RANGE: case FW_EDGE_INPUT_PORT_ALREADY_CONNECTED: *err_node = dst; break;
            default: *err_node = FW_ID_DANGLING;
        }
    }
    if (err_port) *err_port = rc == FW_EDGE_OUT_PORT_OUT_OF_RANGE ? sp : dp;
    return rc;
}
int fw_graph_disconnect(fw_ctx* c, fw_node_id s, uint32_t sp, fw_node_id d, uint32_t dp) { return c->graph->disconnect(Id::unpack(s), sp, Id::unpack(d), dp); }
int fw_graph_disconnect_by_edge_id(fw_ctx* c, fw_edge_id e) { return c->graph->disconnect_edge(Id::unpack(e)); }
int fw_graph_edge(fw_ctx* c, fw_edge_id e, fw_edge_info* out) {
    const EdgeRec* r = c->graph->edge(Id::unpack(e));
    if (!r) return 0;
    if (out) *out = fw_edge_info{r->id.pack(), r->src.pack(), r->dst.pack(), r->src_port, r->dst_port};
    return 1;
}
int fw_graph_node_info(fw_ctx* c, fw_node_id node, fw_node_info* out) {
    NodeRec* r = c->graph->node(Id::unpack(node));
    if (!r) return 0;
    if (out) {
        std::memset(out, 0, sizeof(*out));
        out->num_inputs = r->num_inputs; out->num_outputs = r->num_outputs; out->kind = r->params->kind;
        const NodeKind& nk = node_kind(r->params->kind);
        const fw_audio_node_info& ai = r->params->custom ? r->params->custom->info : nk.info;
        out->num_min_supported_inputs = ai.num_min_supported_inputs; out->num_max_supported_inputs = ai.num_max_supported_inputs;
        out->num_min_supported_outputs = ai.num_min_supported_outputs; out->num_max_supported_outputs = ai.num_max_supported_outputs;
        out->updates = ai.updates != 0;
        const char* name = r->id == c->graph->graph_in() ? "graph_in" : r->id == c->graph->graph_out() ? "graph_out" :
                           r->params->custom ? r->params->custom->debug_name.c_str() : nk.name;
        std::strncpy(out->debug_name, name, sizeof(out->debug_name) - 1);
    }
    return 1;
}
uint32_t fw_graph_num_nodes(fw_ctx* c) { return c->graph->num_nodes(); }
uint32_t fw_graph_num_edges(fw_ctx* c) { return c->graph->num_edges(); }
uint32_t fw_graph_nodes(fw_ctx* c, fw_node_id* out, uint32_t cap) { uint32_t n = 0; c->graph->each_node([&](Id id, NodeRec&) { if (out && n < cap) out[n] = id.pack(); ++n; }); return n; }
uint32_t fw_graph_edges(fw_ctx* c, fw_edge_id* out, uint32_t cap) { uint32_t n = 0; c->graph->each_edge([&](Id id, EdgeRec&) { if (out && n < cap) out[n] = id.pack(); ++n; }); return n; }
int fw_graph_cycle_detected(fw_ctx* c) { return c->graph->cycle_detected(); }
void fw_graph_reset(fw_ctx* c) { c->graph->reset(); }
int fw_graph_needs_compile(fw_ctx* c) { return c->graph->needs_compile(); }

int fw_graph_compile_internal(fw_ctx* c, uint32_t mbf) {
    c->dbg_valid = false;
    if (mbf == 0) return FW_COMPILE_NODE_ACTIVATION_FAILED;
    CompileError e = c->graph->compile_schedule(mbf, &c->dbg_schedule);
    c->dbg_valid = e.code == FW_COMPILE_OK;
    return e.code;
}
uint32_t fw_schedule_len(fw_ctx* c) { return c->dbg_valid ? (uint32_t)c->dbg_schedule.nodes.size() : 0; }
uint32_t fw_schedule_num_buffers(fw_ctx* c) { return c->dbg_valid ? c->dbg_schedule.num_buffers : 0; }
int fw_schedule_node(fw_ctx* c, uint32_t i, fw_scheduled_node* out) {
    if (!c->dbg_valid || i >= c->dbg_schedule.nodes.size() || !out) return 0;
    const SchedNode& sn = c->dbg_schedule.nodes[i];
    std::memset(out, 0, sizeof(*out));
    out->id = sn.id.pack(); out->num_inputs = (uint32_t)sn.in.size(); out->num_outputs = (uint32_t)sn.out.size();
    for (size_t k = 0; k < sn.in.size() && k < 64; ++k) { out->in_buffer[k] = sn.in[k].buffer; out->in_should_clear[k] = sn.in[k].should_clear; }
    for (size_t k = 0; k < sn.out.size() && k < 64; ++k) out->out_buffer[k] = sn.out[k].buffer;
    return 1;
}

// ---- isomorphic-voice detection (SURVEY §8 f2; voices.cpp) ---------------------------------------------------------------------
int fw_graph_detect_voices(fw_ctx* c, fw_voice_template* out) {
    if (!c) return -1;
    auto det = std::make_unique<VoiceDetection>();
    std::string why;
    c->voices.reset();
    if (out) std::memset(out, 0, sizeof(*out));
    if (c->cfg.num_voices != 1) { c->last_error = "detect_voices works on a flat graph (num_voices == 1)"; return -1; }
    if (!detect_voices(*c->graph, det.get(), &why)) { c->last_error = "not a batch of isomorphic voices: " + why; return -1; }
    if (out) { out->num_voices = det->num_voices; out->num_template_nodes = (uint32_t)det->nodes.size(); out->voice_inputs = det->voice_inputs;
               out->voice_outputs = det->voice_outputs; out->num_tree_nodes = (uint32_t)det->tree.size(); }
    c->last_error = why.empty() ? std::string() : "fewer voices than the SumNode tree has leaves: " + why;
    c->voices = std::move(det);
    return 0;
}
uint32_t fw_graph_voice_nodes(fw_ctx* c, uint32_t template_node, fw_node_id* out, uint32_t cap) {
    if (!c || !c->voices || template_node >= c->voices->nodes.size()) return 0;
    const std::vector<Id>& v = c->voices->nodes[template_node];
    for (size_t i = 0; i < v.size() && i < cap && out; ++i) out[i] = v[i].pack();
    return (uint32_t)v.size();
}
// The batched context of a detected flat graph: one voice graph (the template, canonical order), num_voices = V, the per-voice
// parameter tables filled from the V copies, master_bus = 1 in place of the SumNode tree.
fw_ctx* fw_ctx_new_batched(fw_ctx* flat, int32_t device, uint32_t max_call_frames, fw_node_id* template_ids, uint32_t cap) {
    if (!flat) return nullptr;
    if (!flat->voices) { flat->last_error = "ctx_new_batched: call graph_detect_voices first"; return nullptr; }
    const VoiceDetection& d = *flat->voices;
    const uint32_t V = d.num_voices;
    for (const auto& ids : d.nodes) for (Id id : ids) if (!flat->graph->node(id)) { flat->last_error = "ctx_new_batched: the graph changed since detect_voices"; return nullptr; }
    fw_graph_config cfg = flat->cfg;
    cfg.num_graph_inputs = d.voice_inputs; cfg.num_graph_outputs = d.voice_outputs; cfg.num_voices = V; cfg.master_bus = V > 1 ? 1u : flat->cfg.master_bus;
    cfg.device = device; cfg.max_call_frames = max_call_frames;
    fw_ctx* b = fw_ctx_new(&cfg);
    if (!b) return nullptr;
    if (flat->res) b->res = flat->res;  // sample resources are shared: handles stay valid
    std::vector<Id> ids(d.nodes.size());
    for (size_t i = 0; i < d.nodes.size(); ++i) {
        const NodeRec& r0 = *flat->graph->node(d.nodes[i][0]);
        auto p = std::make_shared<NodeParams>(*r0.params);  // static parameters (stages, delay, IR, tables, threshold) from voice 0
        p->num_voices = V;
        auto gather = [&](std::vector<float> NodeParams::*field, size_t per_voice) {
            if (((*r0.params).*field).empty()) return;
            std::vector<float>& dst = (*p).*field;
            dst.assign((size_t)V * per_voice, 0.0f);
            for (uint32_t v = 0; v < V; ++v) {
                const std::vector<float>& src = (*flat->graph->node(d.nodes[i][v])->params).*field;
                std::copy_n(src.begin(), std::min(per_voice, src.size()), dst.begin() + (size_t)v * per_voice);
            }
        };
        gather(&NodeParams::percent, 1); gather(&NodeParams::raw_gain, 1); gather(&NodeParams::pan, 1); gather(&NodeParams::gain_l, 1); gather(&NodeParams::gain_r, 1);
        gather(&NodeParams::coeffs, (size_t)p->num_stages * coeff_width(p->kind));
        if (p->kind == FW_NODE_SAMPLER) { p->smp_active = false; p->smp_playing.assign(V, 0); p->smp_pending.assign(V, 0); p->smp_pending_epoch.assign(V, 0); }
        ids[i] = b->graph->add_node(r0.num_inputs, r0.num_outputs, std::move(p));
        if (template_ids && i < cap) template_ids[i] = ids[i].pack();
    }
    auto wire = [&](const VoiceDetection::Src& s, Id dst, uint32_t dp) {
        if (s.node == -1) return true;
        const Id src = s.node == -2 ? b->graph->graph_in() : ids[(size_t)s.node];
        Id e; return b->graph->connect(src, s.port, dst, dp, false, &e) == FW_EDGE_OK;
    };
    bool ok = true;
    for (size_t i = 0; i < d.inputs.size(); ++i) for (size_t port = 0; port < d.inputs[i].size(); ++port) ok = ok && wire(d.inputs[i][port], ids[i], (uint32_t)port);
    for (size_t ch = 0; ch < d.outputs.size(); ++ch) ok = ok && wire(d.outputs[ch], b->graph->graph_out(), (uint32_t)ch);
    if (!ok) { flat->last_error = "ctx_new_batched: internal: could not rebuild the voice graph"; fw_ctx_free(b); return nullptr; }
    return b;
}
// main-thread view of a node's parameter tables (volume.rs:24,36 / sampler.rs:167,179 are the reference's per-node getters)
uint32_t fw_node_read_params(fw_ctx* c, fw_node_id node, uint32_t which, float* out, uint32_t cap) {
    NodeRec* r = c ? c->graph->node(Id::unpack(node)) : nullptr;
    if (!r) return 0;
    const NodeParams& p = *r->params;
    const std::vector<float>* src = nullptr;
    switch (which) {
        case FW_PARAM_PERCENT_VOLUME: src = &p.percent; break;
        case FW_PARAM_RAW_GAIN: src = &p.raw_gain; break;
        case FW_PARAM_PAN: src = &p.pan; break;
        case FW_PARAM_GAIN_L: src = &p.gain_l; break;
        case FW_PARAM_GAIN_R: src = &p.gain_r; break;
        case FW_PARAM_COEFFS: src = &p.coeffs; break;
        default: return 0;
    }
    for (size_t i = 0; i < src->size() && i < cap && out; ++i) out[i] = (*src)[i];
    return (uint32_t)src->size();
}

}  // extern "C"
// ---- parameters -----------------------------------------------------------------------------
// One path to the stream side, and it takes no lock (context.rs:61-64, "no mutexes" DESIGN_DOC.md:37): every store lands in the
// node's host arrays (the main thread's view, which seeds the device state at activation) and, once the context is active, also
// travels through the wait-free command ring in program order, stamped with the current event block (fw_ctx_set_event_block;
// 0 = the start of the next call). The stream side applies it as an ordered device store at that block — the reference's relaxed
// atomic store / per-block load (volume.rs:29-32,92). Whole-array setters travel as one CMD_UPLOAD with a snapshot of the array.
static NodeParams* params_of(fw_ctx* c, fw_node_id node, uint32_t kind) {
    NodeRec* r = c->graph->node(Id::unpack(node));
    return (r && r->params->kind == kind) ? r->params.get() : nullptr;
}
static bool voice_ok(const NodeParams* p, uint32_t voice) { return p && (voice == FW_ALL_VOICES || voice < p->num_voices); }
template <class F> static void each_voice_of(NodeParams* p, uint32_t voice, F&& f) {
    if (voice == FW_ALL_VOICES) { for (uint32_t v = 0; v < p->num_voices; ++v) f(v); } else f(voice);
}
static bool push_cmd(fw_ctx* c, const Cmd& m) { return c->active && c->ch && c->ch->cmds.push(m); }
static void drain_to_free(fw_ctx* c) { if (c->ch) { float* q; while (c->ch->to_free.pop(&q)) delete[] q; } }
// store into the main thread's view; once active, the same store travels to the stream side as a command stamped with the
// current event block (0: the start of the next call)
template <class F> static int store_param(fw_ctx* c, NodeParams* p, uint32_t voice, Cmd m, F&& write_host) {
    if (!voice_ok(p, voice)) return -1;
    each_voice_of(p, voice, write_host);
    if (!c->active) return 0;
    m.block = c->event_block; m.voice = voice; m.node = p;
    return push_cmd(c, m) ? 0 : -2;  // -2: command ring full
}
// a whole array at once: the snapshot is taken here, uploaded by the stream side in ring order, and handed back for freeing
static int upload_array(fw_ctx* c, NodeParams* p, uint32_t which, const float* data, size_t n) {
    if (!c->active) return 0;
    drain_to_free(c);
    float* snap = new float[n ? n : 1];
    std::memcpy(snap, data, n * sizeof(float));
    Cmd m{}; m.kind = CMD_UPLOAD; m.block = c->event_block; m.voice = FW_ALL_VOICES; m.a = which; m.x = reinterpret_cast<uint64_t>(snap); m.y = n; m.node = p;
    if (!push_cmd(c, m)) { delete[] snap; return -2; }
    return 0;
}
// `(secs * sample_rate).round() as u64` (sampler.rs:250-251,394): saturating float -> int cast, NaN -> 0
static uint64_t secs_to_frame(double secs, uint32_t sample_rate) {
    const double f = std::round(secs * (double)sample_rate);
    if (!(f > 0.0)) return 0;
    if (f >= 18446744073709551616.0) return UINT64_MAX;
    return (uint64_t)f;
}
// push one message for the selected voices; `gate(v)` mirrors the node-side `playing` checks (sampler.rs:82-136)
template <class G> static int sampler_push(fw_ctx* c, fw_node_id node, uint32_t voice, uint32_t kind, uint32_t b, uint64_t x, uint64_t y, G&& gate) {
    NodeParams* p = c ? params_of(c, node, FW_NODE_SAMPLER) : nullptr;
    if (!p || (voice != FW_ALL_VOICES && voice >= p->num_voices)) return FW_SAMPLER_NOT_A_SAMPLER;
    if (!p->smp_active || !c->active) return FW_SAMPLER_NOT_ACTIVATED;
    int rc = FW_SAMPLER_OK;
    const uint32_t epoch = c->ch->drain_epoch.load(std::memory_order_acquire);
    const uint32_t v0 = voice == FW_ALL_VOICES ? 0 : voice, v1 = voice == FW_ALL_VOICES ? p->num_voices : voice + 1;
    bool all = voice == FW_ALL_VOICES;
    // per-voice ring capacity 128 (sampler.rs:14): count what was queued since the stream side last drained
    for (uint32_t v = v0; v < v1; ++v) {
        if (p->smp_pending_epoch[v] != epoch) { p->smp_pending_epoch[v] = epoch; p->smp_pending[v] = 0; }
        if (!gate(*p, v, /*probe=*/true) || p->smp_pending[v] >= 128) all = false;
    }
    Cmd m{}; m.kind = CMD_SAMPLER; m.block = c->event_block; m.a = kind; m.b = b; m.x = x; m.y = y; m.node = p;
    if (all) {  // one command for every voice
        m.voice = FW_ALL_VOICES;
        if (!push_cmd(c, m)) return FW_SAMPLER_RING_FULL;
        for (uint32_t v = v0; v < v1; ++v) { p->smp_pending[v]++; gate(*p, v, /*probe=*/false); }
        return rc;
    }
    for (uint32_t v = v0; v < v1; ++v) {
        if (!gate(*p, v, /*probe=*/true)) continue;
        if (p->smp_pending[v] >= 128) { rc = FW_SAMPLER_RING_FULL; continue; }  // rtrb push Err
        m.voice = v;
        if (!push_cmd(c, m)) { rc = FW_SAMPLER_RING_FULL; continue; }
        p->smp_pending[v]++; gate(*p, v, /*probe=*/false);
    }
    return rc;
}
static bool gate_always(NodeParams&, uint32_t, bool) { return true; }
extern "C" {
void fw_ctx_set_event_block(fw_ctx* c, uint32_t block) { if (c) c->event_block = block; }
// ---- biquad / SVF coefficient table: [voice][stage][coeff_width(kind)] ------------------------
static int set_stage_coeffs(fw_ctx* c, fw_node_id node, uint32_t kind, uint32_t voice, uint32_t stage, const float* k) {
    NodeParams* p = params_of(c, node, kind);
    if (!p || !k || stage >= p->num_stages) return -1;
    const uint32_t w = coeff_width(kind);
    Cmd m{}; m.kind = CMD_COEFFS; m.a = stage; std::memcpy(m.f, k, w * sizeof(float));
    return store_param(c, p, voice, m, [&](uint32_t v) { std::memcpy(&p->coeffs[((size_t)v * p->num_stages + stage) * w], k, w * sizeof(float)); });
}
static int set_all_coeffs(fw_ctx* c, fw_node_id node, uint32_t kind, const float* k, uint32_t nv, uint32_t ns) {
    NodeParams* p = params_of(c, node, kind);
    if (!p || !k || nv != p->num_voices || ns != p->num_stages) return -1;
    std::memcpy(p->coeffs.data(), k, (size_t)nv * ns * coeff_width(kind) * sizeof(float));
    return upload_array(c, p, 2, p->coeffs.data(), p->coeffs.size());
}
// ---- SVF + polyphase resampler (spec ours) ----------------------------------------------------
int fw_svf_set_coeffs(fw_ctx* c, fw_node_id node, uint32_t voice, uint32_t stage, const float* k) { return set_stage_coeffs(c, node, FW_NODE_SVF, voice, stage, k); }
int fw_svf_set_all_coeffs(fw_ctx* c, fw_node_id node, const float* k, uint32_t nv, uint32_t ns) { return set_all_coeffs(c, node, FW_NODE_SVF, k, nv, ns); }
void fw_svf_design(uint32_t type, double fc, double q, double sr, float* out) {
    const double g = std::tan(M_PI * fc / sr), k = 1.0 / q;
    const double a1 = 1.0 / (1.0 + g * (g + k)), a2 = g * a1, a3 = g * a2;
    double m0 = 0, m1 = 0, m2 = 1;
    switch (type) {
        case 1: m0 = 0; m1 = 1; m2 = 0; break;
        case 2: m0 = 1; m1 = -k; m2 = -1; break;
        case 3: m0 = 1; m1 = -k; m2 = 0; break;
        case 4: m0 = 1; m1 = -k; m2 = -2; break;
        case 5: m0 = 1; m1 = -2 * k; m2 = 0; break;
        default: break;
    }
    out[0] = (float)a1; out[1] = (float)a2; out[2] = (float)a3; out[3] = (float)m0; out[4] = (float)m1; out[5] = (float)m2;
}
// resampler transport travels as commands (event block 0: the start of the next call); before activation nothing can play
int fw_resampler_set(fw_ctx* c, fw_node_id node, uint32_t voice, uint32_t res, uint64_t step, int playing, int loop) {
    NodeParams* p = c ? params_of(c, node, FW_NODE_RESAMPLER) : nullptr;
    uint64_t frames = 0;
    if (!voice_ok(p, voice) || (res != 0 && (!c->res || !c->res->frames_of(res, &frames)))) return -1;
    Cmd m{}; m.kind = CMD_RS_SET; m.block = c->event_block; m.voice = voice; m.a = (playing ? 1u : 0u) | (loop ? 2u : 0u); m.b = res; m.x = step; m.node = p;
    return push_cmd(c, m) ? 0 : -2;
}
int fw_resampler_seek(fw_ctx* c, fw_node_id node, uint32_t voice, uint64_t pos_frames) {
    NodeParams* p = c ? params_of(c, node, FW_NODE_RESAMPLER) : nullptr;
    if (!voice_ok(p, voice)) return -1;
    Cmd m{}; m.kind = CMD_RS_SEEK; m.block = c->event_block; m.voice = voice; m.x = pos_frames; m.node = p;
    return push_cmd(c, m) ? 0 : -2;
}
static double bessel_i0(double x) { double s = 1.0, t = 1.0; for (int k = 1; k < 64; ++k) { t *= (x / (2.0 * k)) * (x / (2.0 * k)); s += t; if (t < 1e-18 * s) break; } return s; }
void fw_resampler_design(uint32_t P, uint32_t T, double cutoff, double beta, float* table) {
    const double half = (double)T / 2.0, i0b = bessel_i0(beta);
    for (uint32_t ph = 0; ph < P; ++ph) for (uint32_t t = 0; t < T; ++t) {
        const double x = (double)t - (half - 1.0) - (double)ph / (double)P;
        const double sn = x == 0.0 ? 1.0 : std::sin(M_PI * cutoff * x) / (M_PI * cutoff * x);
        const double r = x / half, w = std::fabs(r) >= 1.0 ? 0.0 : bessel_i0(beta * std::sqrt(1.0 - r * r)) / i0b;
        table[(size_t)ph * T + t] = (float)(cutoff * sn * w);
    }
}

// ---- sample resources + SamplerNode (sampler.rs:46-181) --------------------------------------
uint32_t fw_sample_resource_create(fw_ctx* c, uint32_t format, uint32_t channels, uint64_t frames, const void* data) {
    if (!c || !data || format > FW_SAMPLE_U16_PLANAR || channels == 0 || channels > 64 || frames == 0) return 0;
    if (!c->res) c->res = std::make_shared<ResTable>(c->cfg.device);
    return c->res->add(format, channels, frames, data);
}
int fw_sampler_set_sample(fw_ctx* c, fw_node_id node, uint32_t voice, uint32_t res, int stop_playback) {
    uint64_t frames = 0;
    if (!c || !c->res || !c->res->frames_of(res, &frames)) return FW_SAMPLER_BAD_ARGS;
    return sampler_push(c, node, voice, SMSG_SET_SAMPLE, res, stop_playback ? 1ull : 0ull, 0, gate_always);
}
int fw_sampler_play(fw_ctx* c, fw_node_id node, uint32_t voice) {
    return sampler_push(c, node, voice, SMSG_PLAY, 0, 0, 0,
                        [](NodeParams& p, uint32_t v, bool probe) { if (probe) return !p.smp_playing[v]; p.smp_playing[v] = 1; return true; });
}
int fw_sampler_pause(fw_ctx* c, fw_node_id node, uint32_t voice) {
    return sampler_push(c, node, voice, SMSG_PAUSE, 0, 0, 0,
                        [](NodeParams& p, uint32_t v, bool probe) { if (probe) return (bool)p.smp_playing[v]; p.smp_playing[v] = 0; return true; });
}
int fw_sampler_stop(fw_ctx* c, fw_node_id node, uint32_t voice) {
    return sampler_push(c, node, voice, SMSG_STOP, 0, 0, 0,
                        [](NodeParams& p, uint32_t v, bool probe) { if (probe) return (bool)p.smp_playing[v]; p.smp_playing[v] = 0; return true; });
}
int fw_sampler_set_playhead(fw_ctx* c, fw_node_id node, uint32_t voice, double secs) {
    if (!c) return FW_SAMPLER_NOT_A_SAMPLER;
    return sampler_push(c, node, voice, SMSG_SET_PLAYHEAD, 0, secs_to_frame(secs, c->sample_rate), 0, gate_always);
}
int fw_sampler_set_loop_range(fw_ctx* c, fw_node_id node, uint32_t voice, uint32_t mode, double s, double e) {
    if (!c || mode > FW_LOOP_RANGE_SECS) return FW_SAMPLER_BAD_ARGS;
    const uint64_t fs = mode == FW_LOOP_RANGE_SECS ? secs_to_frame(s, c->sample_rate) : 0, fe = mode == FW_LOOP_RANGE_SECS ? secs_to_frame(e, c->sample_rate) : 0;
    if (mode == FW_LOOP_RANGE_SECS && c->active && !(fs < fe)) return FW_SAMPLER_BAD_ARGS;
    return sampler_push(c, node, voice, SMSG_SET_LOOP, mode, fs, fe, gate_always);
}
static int set_raw_gain(fw_ctx* c, NodeParams* p, uint32_t voice, float pct) {  // volume.rs:28-34, range.rs:32-35 / sampler.rs:174-180
    const float n = std::fmax(pct, 0.0f) * (1.0f / 100.0f), g = n * n;
    Cmd m{}; m.kind = CMD_TARGET; m.a = 0; m.f[0] = g;
    return store_param(c, p, voice, m, [&](uint32_t v) { p->raw_gain[v] = g; p->percent[v] = std::fmax(pct, 0.0f); });
}
int fw_sampler_set_percent_volume(fw_ctx* c, fw_node_id node, uint32_t voice, float pct) {
    NodeParams* p = c ? params_of(c, node, FW_NODE_SAMPLER) : nullptr;
    return set_raw_gain(c, p, voice, pct) == 0 ? FW_SAMPLER_OK : FW_SAMPLER_NOT_A_SAMPLER;
}
int fw_sampler_is_playing(fw_ctx* c, fw_node_id node, uint32_t voice) {
    NodeParams* p = c ? params_of(c, node, FW_NODE_SAMPLER) : nullptr;
    if (!p || voice >= p->num_voices) return FW_SAMPLER_NOT_A_SAMPLER;
    return p->smp_playing[voice] ? 1 : 0;
}

int fw_volume_set_percent_volume(fw_ctx* c, fw_node_id node, uint32_t voice, float pct) { return set_raw_gain(c, params_of(c, node, FW_NODE_VOLUME), voice, pct); }
int fw_volume_set_percent_volumes(fw_ctx* c, fw_node_id node, const float* pct, uint32_t n) {
    NodeParams* p = params_of(c, node, FW_NODE_VOLUME);
    if (!p || n != p->num_voices) return -1;
    for (uint32_t v = 0; v < n; ++v) { float x = std::fmax(pct[v], 0.0f) * (1.0f / 100.0f); p->raw_gain[v] = x * x; p->percent[v] = std::fmax(pct[v], 0.0f); }
    return upload_array(c, p, 0, p->raw_gain.data(), n);
}
static void pan_gains(float pan, float* gl, float* gr) {
    double pp = std::fmin(std::fmax((double)pan, -1.0), 1.0), th = (pp + 1.0) * (M_PI / 4.0);
    *gl = (float)std::cos(th); *gr = (float)std::sin(th);
}
static int set_pan_gains(fw_ctx* c, NodeParams* p, uint32_t voice, float gl, float gr, const float* pan) {
    if (!voice_ok(p, voice)) return -1;
    each_voice_of(p, voice, [&](uint32_t v) { p->gain_l[v] = gl; p->gain_r[v] = gr; if (pan) p->pan[v] = *pan; });
    if (!c->active) return 0;
    Cmd m{}; m.kind = CMD_TARGET; m.block = c->event_block; m.voice = voice; m.node = p;
    m.a = 0; m.f[0] = gl; const bool ok0 = push_cmd(c, m);
    m.a = 1; m.f[0] = gr; const bool ok1 = push_cmd(c, m);
    return ok0 && ok1 ? 0 : -2;
}
int fw_pan_set_pan(fw_ctx* c, fw_node_id node, uint32_t voice, float pan) {
    float gl, gr; pan_gains(pan, &gl, &gr);
    return set_pan_gains(c, params_of(c, node, FW_NODE_PAN), voice, gl, gr, &pan);
}
int fw_pan_set_pans(fw_ctx* c, fw_node_id node, const float* pan, uint32_t n) {
    NodeParams* p = params_of(c, node, FW_NODE_PAN);
    if (!p || n != p->num_voices) return -1;
    for (uint32_t v = 0; v < n; ++v) { p->pan[v] = pan[v]; pan_gains(pan[v], &p->gain_l[v], &p->gain_r[v]); }
    const int r0 = upload_array(c, p, 0, p->gain_l.data(), n), r1 = upload_array(c, p, 1, p->gain_r.data(), n);
    return r0 ? r0 : r1;
}
int fw_pan_set_gains(fw_ctx* c, fw_node_id node, uint32_t voice, float gl, float gr) { return set_pan_gains(c, params_of(c, node, FW_NODE_PAN), voice, gl, gr, nullptr); }
int fw_biquad_set_coeffs(fw_ctx* c, fw_node_id node, uint32_t voice, uint32_t stage, const float* k) { return set_stage_coeffs(c, node, FW_NODE_BIQUAD, voice, stage, k); }
int fw_biquad_set_all_coeffs(fw_ctx* c, fw_node_id node, const float* k, uint32_t nv, uint32_t ns) { return set_all_coeffs(c, node, FW_NODE_BIQUAD, k, nv, ns); }
void fw_biquad_design_rbj(uint32_t type, double fc, double q, double gain_db, double sr, float* out) {  // RBJ cookbook, f64 -> f32
    const double w0 = 2.0 * M_PI * fc / sr, cw = std::cos(w0), sw = std::sin(w0), alpha = sw / (2.0 * q), A = std::pow(10.0, gain_db / 40.0);
    double b0, b1, b2, a0, a1, a2;
    switch (type) {
        case 0: b0 = (1 - cw) / 2; b1 = 1 - cw; b2 = (1 - cw) / 2; a0 = 1 + alpha; a1 = -2 * cw; a2 = 1 - alpha; break;
        case 1: b0 = (1 + cw) / 2; b1 = -(1 + cw); b2 = (1 + cw) / 2; a0 = 1 + alpha; a1 = -2 * cw; a2 = 1 - alpha; break;
        case 2: b0 = alpha; b1 = 0; b2 = -alpha; a0 = 1 + alpha; a1 = -2 * cw; a2 = 1 - alpha; break;
        case 3: b0 = 1; b1 = -2 * cw; b2 = 1; a0 = 1 + alpha; a1 = -2 * cw; a2 = 1 - alpha; break;
        case 4: b0 = 1 + alpha * A; b1 = -2 * cw; b2 = 1 - alpha * A; a0 = 1 + alpha / A; a1 = -2 * cw; a2 = 1 - alpha / A; break;
        case 5: { const double s = 2 * std::sqrt(A) * alpha;
            b0 = A * ((A + 1) - (A - 1) * cw + s); b1 = 2 * A * ((A - 1) - (A + 1) * cw); b2 = A * ((A + 1) - (A - 1) * cw - s);
            a0 = (A + 1) + (A - 1) * cw + s; a1 = -2 * ((A - 1) + (A + 1) * cw); a2 = (A + 1) + (A - 1) * cw - s; break; }
        default: { const double s = 2 * std::sqrt(A) * alpha;
            b0 = A * ((A + 1) + (A - 1) * cw + s); b1 = -2 * A * ((A - 1) + (A + 1) * cw); b2 = A * ((A + 1) + (A - 1) * cw - s);
            a0 = (A + 1) - (A - 1) * cw + s; a1 = 2 * ((A - 1) - (A + 1) * cw); a2 = (A + 1) - (A - 1) * cw - s; break; }
    }
    out[0] = (float)(b0 / a0); out[1] = (float)(b1 / a0); out[2] = (float)(b2 / a0); out[3] = (float)(a1 / a0); out[4] = (float)(a2 / a0);
}

// ---- lifecycle --------------------------------------------------------------------------------
int fw_ctx_activate(fw_ctx* c, uint32_t sr, uint32_t n_in, uint32_t n_out, uint32_t mbf, void* user_cx, fw_processor** out) {
    if (!c || !out || sr == 0 || mbf == 0 || n_in > 64 || n_out > 64) { if (c) c->last_error = "bad activate arguments"; return -1; }
    if (c->active) return 1;  // context.rs:57-59
    int ndev = 0;
    if (!FW_CUDA(cudaGetDeviceCount(&ndev)) || c->cfg.device < 0 || c->cfg.device >= ndev) {
        c->last_error = "no CUDA device " + std::to_string(c->cfg.device) + " (firewheel-b200 has no CPU fallback): " + g_dev_err;
        return -1;
    }
    if (!FW_CUDA(cudaSetDevice(c->cfg.device))) { c->last_error = g_dev_err; return -1; }
    auto p = std::make_unique<fw_processor>(c->cfg.device);  // the context turns active only once the processor is complete
    bool ok = FW_CUDA(cudaStreamCreateWithFlags(&p->stream, cudaStreamNonBlocking));
    for (int i = 0; ok && i < 4; ++i) ok = FW_CUDA(cudaEventCreate(&p->ev[i]));
    p->h_masks = p->mem.host<uint64_t>(c->cfg.num_voices + 1); p->h_err = p->mem.host<uint32_t>(1);
    if (!ok || !p->mem.ok()) { c->last_error = g_dev_err; return -1; }
    p->bus = c->cfg.master_bus != 0;
    const uint32_t max_call = c->cfg.max_call_frames ? c->cfg.max_call_frames : 64u * mbf;
    p->max_call_frames = ((max_call + mbf - 1) / mbf) * mbf;  // whole blocks
    {
        const size_t V = c->cfg.num_voices, Tm = p->max_call_frames;
        const size_t in_e = V * n_in * Tm, out_e = (size_t)(p->bus ? 1 : V) * n_out * Tm;
        p->d_in = p->mem.dev<float>(in_e, false); p->d_out = p->mem.dev<float>(out_e, false); p->d_inter = p->mem.dev<float>(std::max(in_e, out_e), false);
        if (!p->mem.ok()) { c->last_error = "device allocation failed (I/O staging for max_call_frames): " + g_dev_err; return -1; }
    }
    c->ch = std::make_shared<Channels>(std::max<size_t>(4096, 4 * (size_t)c->cfg.num_voices));
    c->active = true; c->sample_rate = sr; c->max_block_frames = mbf; c->n_in = n_in; c->n_out = n_out; c->max_call_frames = p->max_call_frames;
    p->ch = c->ch; p->user_cx = user_cx; p->num_voices = c->cfg.num_voices; p->max_block_frames = mbf; p->n_in = n_in; p->n_out = n_out;
    p->pend.resize(2 * c->ch->cmds.capacity()); p->cmd_ptrs.resize(p->pend.size());
    // SmootherConfig::default + ParamSmoother::new (smoother.rs:18-25,99-100); host libm, once
    p->sm_b = std::exp(-1.0f / ((10.0f / 1000.0f) * (float)sr)); p->sm_a = 1.0f - p->sm_b; p->sm_eps = 0.00001f;
    *out = p.release();
    return 0;
}
int fw_ctx_is_activated(fw_ctx* c) { return c->active; }

int fw_ctx_update(fw_ctx* c, fw_update_status* out) {  // context.rs:93-148
    fw_update_status st{}; st.kind = FW_UPDATE_INACTIVE; st.error_node = FW_ID_DANGLING;
    auto done = [&] { if (out) *out = st; return 0; };
    drain_to_free(c);
    c->graph->each_node([&](Id, NodeRec& r) {  // self.graph.update() (context.rs:94, graph.rs:691-697)
        if (r.params->custom && r.params->custom->info.updates && r.params->custom->vt.update) r.params->custom->vt.update(r.params->custom->node);
    });
    if (!c->active) return done();
    bool dropped = false; void* cx = nullptr;
    ctx_drain(c, &dropped, &cx);
    if (dropped) { ctx_graph_deactivate(c); c->active = false; c->ch.reset(); st.kind = FW_UPDATE_DEACTIVATED; st.returned_user_cx = cx; return done(); }
    st.kind = FW_UPDATE_ACTIVE;
    if (!c->graph->needs_compile()) return done();
    cudaSetDevice(c->cfg.device);
    auto plan = std::make_unique<Plan>(c->cfg.device);
    CompileError e = c->graph->compile_schedule(c->max_block_frames, &plan->sched);
    if (e.code != FW_COMPILE_OK) { st.graph_error = e.code; st.error_node = e.node.pack(); st.error_port = e.port; return done(); }
    // A live node whose port count changed (set_num_inputs / set_num_outputs, graph.rs:315-393) no longer matches the per-channel
    // state its device counterpart was sized for: it is activated again with the new counts (fresh state), the old state leaves
    // with the outgoing plan.
    c->graph->each_node([&](Id id, NodeRec& r) {
        auto it = c->node_states.find(id.pack());
        if (it == c->node_states.end()) return;
        if (node_kind(it->second->kind).per_channel_state && it->second->channels != r.num_inputs) {
            c->node_states.erase(it);
            if (std::find(c->graph->nodes_to_activate.begin(), c->graph->nodes_to_activate.end(), id) == c->graph->nodes_to_activate.end()) c->graph->nodes_to_activate.push_back(id);
        }
    });
    // activate new nodes in queue order (graph.rs:593-612); a failure rolls back this round's activations
    std::vector<uint64_t> created;
    for (Id id : c->graph->nodes_to_activate) {
        NodeRec* r = c->graph->node(id);
        if (!r) continue;
        std::string msg = node_check_activation(*r->params, r->num_inputs, r->num_outputs);
        std::shared_ptr<NodeDeviceState> ds;
        if (msg.empty()) {
            ds = std::make_shared<NodeDeviceState>(c->cfg.device);
            ds->kind = r->params->kind; ds->V = c->cfg.num_voices; ds->params = r->params; ds->channels = r->num_inputs;
            if (r->params->custom) {  // AudioNode::activate (node.rs:12-18)
                char err[256] = {0};
                void* proc_h = nullptr;
                const int arc = r->params->custom->vt.activate(r->params->custom->node, c->sample_rate, c->max_block_frames, r->num_inputs, r->num_outputs, c->cfg.num_voices,
                                                              c->cfg.device, &proc_h, err, (uint32_t)sizeof(err) - 1);
                if (arc != 0 || !proc_h) msg = err[0] ? std::string(err) : std::string("custom node activation failed");
                else {
                    ds->custom_proc = proc_h;
                }
            }
            if (node_kind(ds->kind).reads_resources && !c->res) c->res = std::make_shared<ResTable>(c->cfg.device);
            if (!ds->create()) msg = "device allocation failed: " + g_dev_err;
        }
        if (!msg.empty()) {
            if (ds && ds->custom_proc) ds->custom_deactivate = true;
            for (uint64_t k : created) { auto it = c->node_states.find(k); if (it != c->node_states.end()) { it->second->custom_deactivate = true; c->node_states.erase(it); } }  // roll-back: deactivate(Some(processor)) (graph.rs:603-609)
            st.graph_error = FW_COMPILE_NODE_ACTIVATION_FAILED; st.error_node = id.pack(); c->last_error = msg;
            return done();
        }
        c->node_states[id.pack()] = ds; created.push_back(id.pack());
    }
    std::string why;
    if (!lower(c, plan->sched, plan.get(), &why)) {
        for (uint64_t k : created) { auto it = c->node_states.find(k); if (it != c->node_states.end()) { it->second->custom_deactivate = true; c->node_states.erase(it); } }
        st.graph_error = FW_COMPILE_UNSUPPORTED_ON_DEVICE; c->last_error = why;
        return done();
    }
    plan->nodes_to_remove = c->graph->nodes_removed_since_compile;
    for (Id id : plan->nodes_to_remove) {  // the outgoing plan still holds them until it is returned; then deactivate(Some(processor)) (graph.rs:644-648)
        auto it = c->node_states.find(id.pack());
        if (it != c->node_states.end()) { it->second->custom_deactivate = true; c->node_states.erase(it); }
    }
    c->graph->clear_dirty(); c->graph->nodes_to_activate.clear(); c->graph->nodes_removed_since_compile.clear();
    cudaDeviceSynchronize();  // tables and initial state are resident before the stream side can see the plan
    CtxToProc m; m.kind = 0; m.plan = plan.get();
    if (c->ch->to_proc.push(m)) plan.release();
    else std::fprintf(stderr, "firewheel-b200: failed to send new schedule: message channel is full\n");  // context.rs:128-136
    return done();
}

void* fw_ctx_deactivate(fw_ctx* c, int stream_is_running) {  // context.rs:162-211
    if (!c->active) return nullptr;
    using clock = std::chrono::steady_clock;
    const auto start = clock::now();
    bool dropped = false; void* cx = nullptr;
    if (stream_is_running) {
        CtxToProc m; m.kind = 1;
        while (!c->ch->to_proc.push(m)) {
            std::this_thread::sleep_for(std::chrono::milliseconds(2));
            if (clock::now() - start > std::chrono::seconds(3)) { dropped = true; break; }
        }
    }
    while (!dropped) {
        ctx_drain(c, &dropped, &cx);
        if (!dropped) {
            std::this_thread::sleep_for(std::chrono::milliseconds(2));
            if (clock::now() - start > std::chrono::seconds(3)) dropped = true;
        }
    }
    if (c->ch.use_count() == 1) { CtxToProc m; while (c->ch->to_proc.pop(&m)) delete m.plan; }  // the processor is gone: schedules it never adopted are released here
    ctx_graph_deactivate(c);
    c->active = false; c->ch.reset();
    return cx;
}

// ---- stream side --------------------------------------------------------------------------------
// make the main stream wait for an outstanding master-bus exchange (side stream)
static void join_side(fw_processor* p) {
    for (int q = 0; q < 2; ++q) if (p->exchange_pending[q]) { cudaStreamWaitEvent(p->stream, p->ev_exchange_done[q], 0); p->exchange_pending[q] = false; }
}

static void proc_poll(fw_processor* p) {  // processor.rs:167-206
    CtxToProc m;
    while (p->ch->to_proc.pop(&m)) {
        if (m.kind == 1) { p->running = false; continue; }
        if (p->plan) {
            ProcToCtx r; r.kind = 0; r.plan = p->plan;
            cudaStreamSynchronize(p->stream);  // the old plan's buffers may still be in flight
            if (p->side) cudaStreamSynchronize(p->side);
            p->ch->to_ctx.push(r);
            p->pending_zero_first = true;  // Q11: the swap happens after this block's inputs were written to the old pool
        }
        p->plan = m.plan;
        for (auto& g : p->graphs) { if (g.exec) cudaGraphExecDestroy(g.exec); g = fw_processor::GraphEntry{}; }  // captured sequences point into the old plan
    }
}
// One chunk of a call: frames [t0, t0 + Tc) of rows that are Tfull frames long in the caller's buffers. res_tab / n_res: the snapshot of
// the plan's resource table that every sampler and resampler reads in this chunk (see proc_call).
struct Chunk { uint32_t t0, Tc, Tfull, zero_first; const ResDesc* res_tab; uint32_t n_res; };

// One chain-kernel launch of `prog` over the chunk: channel c of voice v is read at in[c] + v * in_vs and written at out[c] + v * out_vs
// (floats); an unused second channel repeats channel 0, and the bus stage reads all `prog.c_in` (up to kMaxBusChannels). `caller`: `in`
// is the caller's rows, whose first block reads as zero after a schedule swap (Q11); otherwise it is the output of the preceding kernel,
// which the launch waits for.
static ChainArgs chain_args(const Plan& pl, const Chunk& ck, const ChainProgram& prog, const float* const* in, uint64_t in_vs, float* const* out,
                            uint64_t out_vs, bool caller) {
    ChainArgs xa{};
    for (uint32_t c = 0; c < prog.c_in; ++c) xa.in_ch[c] = in[c];
    if (prog.c_in & 1u) xa.in_ch[prog.c_in] = in[prog.c_in - 1];  // an odd last channel is read as a pair with itself
    xa.in_vstride = in_vs;
    xa.out_ch[0] = out[0]; xa.out_ch[1] = out[prog.c_out > 1 ? 1 : 0]; xa.out_vstride = out_vs;
    xa.num_voices = pl.num_voices; xa.frames = ck.Tc; xa.block_frames = pl.block_frames; xa.zero_first_block = (caller && ck.zero_first) ? 1u : 0u;
    xa.in_from_prev_kernel = caller ? 0u : 1u; xa.rec = pl.rec; xa.prog = prog;
    return xa;
}

// Last stage with a master bus: the chain kernel (BUS variant) reduces 64 voices per CTA into partial buses, the combine
// kernel finishes the tree, and with several ranks the per-rank buses are exchanged (SURVEY §8e). bus_out = the caller's
// bus rows (pitch ck.Tfull) at the chunk's first frame.
static int run_bus_stage(fw_processor* p, Plan& pl, ChainArgs& xa, uint32_t n_out, const Chunk& ck, float* bus_out) {
    const uint32_t V = p->num_voices, T = ck.Tc;
    uint32_t n = chain_voice_groups(V);
    // this rank's bus: with several ranks it is gathered and tree-summed below, else it is the caller's bus
    const int q = (int)((p->xepoch + 1u) & 1u);
    float* bus_dst = p->world > 1 ? p->d_bus_local[q] : bus_out;
    const uint32_t bus_pitch = p->world > 1 ? T : ck.Tfull;
    if (p->world > 1 && p->exchange_pending[q]) {
        // buffer q was last read by the exchange two calls back: long done in any steady loop. Only if the side stream really lags is
        // an event wait put on the main stream (it would cut the PDL chain).
        if (cudaEventQuery(p->ev_exchange_done[q]) != cudaSuccess) { cudaGetLastError(); cudaStreamWaitEvent(p->stream, p->ev_exchange_done[q], 0); }
        p->exchange_pending[q] = false;
    }
    if (n == 1) { xa.out = bus_dst; xa.bus_pitch = bus_pitch; }
    else { xa.out = pl.d_part[0]; xa.bus_pitch = 0; }
    if (!FW_LAUNCH(p, 1, 1, launch_chain(xa, true, p->stream))) return FW_PROC_DEVICE_ERROR;
    // With several ranks and the exchange on the side stream, the kernel that completes the rank-local bus also publishes the exchange
    // epoch (last CTA done -> device word): the main stream then has exactly the kernels of the single-GPU case.
    const bool in_line = pl.heavy_stage;
    const bool hand_over = p->world > 1 && !in_line;
    const uint32_t e = p->world > 1 ? ++p->xepoch : 0u;
    bool signalled = false;
    ProfScope ps2(p, 2);
    int cur = 0;
    while (n > 1) {
        const uint32_t n_next = (n + 15) / 16;
        float* cdst = n_next == 1 ? bus_dst : pl.d_part[cur ^ 1];
        const bool sig = hand_over && n_next == 1;
        if (!FW_CUDA(launch_combine(pl.d_part[cur], cdst, n, n_out, T, p->stream, n_next == 1 ? bus_pitch : 0, sig ? p->d_handover : nullptr, sig ? p->d_handover + 1 : nullptr, e))) return FW_PROC_DEVICE_ERROR;
        p->launches++;
        signalled = signalled || sig;
        n = n_next; cur ^= 1;
    }
    if (p->world > 1) {
        // Exchange step (SURVEY §8e) on the high-priority side stream, overlapping control + chain of the next call: all-gather the
        // per-rank buses over NVLink (NCCL), then the top log2(world) levels of the same balanced tree in rank order on every rank —
        // bit-identical on all ranks, unlike ncclAllReduce. Main -> side hand-over through a device word (exchange.cu): the main
        // stream carries no event, its programmatic-dependent-launch chain runs straight into the next call.
        // A plan with a FIR-reverb stage keeps every SM occupied by the GEMM's persistent CTAs (197 KB of shared memory each): a
        // side-stream collective cannot become resident next to them and ends up serialised into the gaps. Such plans run the
        // exchange in line.
        cudaStream_t xs = in_line ? p->stream : p->side;
        if (hand_over) {
            if (!signalled) { if (!FW_CUDA(launch_bus_signal(p->d_handover, e, p->stream))) return FW_PROC_DEVICE_ERROR; p->launches++; }  // <= 64 voices: the chain kernel wrote the bus itself
            if (!FW_CUDA(launch_bus_wait(p->d_handover, e, xa.rec.error, (p->call_epoch << 4) | 2u, p->side))) return FW_PROC_DEVICE_ERROR;
            p->launches++;
        }
        if (!g_nccl.ok(g_nccl.AllGather(p->d_bus_local[q], p->d_gather[q], (size_t)n_out * T, /*ncclFloat32*/ 7, p->nccl_comm, xs), "ncclAllGather")) return FW_PROC_DEVICE_ERROR;
        p->launches++;
        if (!FW_CUDA(launch_combine(p->d_gather[q], bus_out, (uint32_t)p->world, n_out, T, xs, ck.Tfull))) return FW_PROC_DEVICE_ERROR;
        p->launches++;
        if (!in_line) { cudaEventRecord(p->ev_exchange_done[q], p->side); p->exchange_pending[q] = true; }
    }
    return FW_PROC_OK;
}

// ---- launches of the stateful node kinds (see enqueue_chunk) ------------------------------------------------------------------
// C channels of every voice: row v * C + k (voice v, channel k) starts at in + row * in_pitch and at out + row * out_pitch floats.
// A step's input and output operand k resolve to block k: a fused-chain stage has one block of all its channels ([V][C][pitch]), the
// generic lowering a block per channel (C = 1): a pool buffer [V][T] or one channel of the caller's rows (pitch = n_in * Tfull).
struct RowBlock { const float* in; float* out; uint32_t C; uint64_t in_pitch, out_pitch; };
static uint32_t channels_of(const RowBlock* b, uint32_t nb) { uint32_t n = 0; for (uint32_t i = 0; i < nb; ++i) n += b[i].C; return n; }

// SamplerNode: one launch writes the output rows of every block.
static int run_sampler(fw_processor* p, const Plan& pl, const Chunk& ck, const NodeDeviceState& st, const SmpRec* srec, int sm, const RowBlock* b, uint32_t nb) {
    SamplerArgs sa{};
    for (uint32_t i = 0; i < nb; ++i) {
        for (uint32_t k = 0; k < b[i].C; ++k) sa.out[sa.n_out++] = b[i].out + k * b[i].out_pitch;
        sa.out_vstride = b[i].C * b[i].out_pitch;
    }
    sa.num_voices = p->num_voices; sa.frames = ck.Tc; sa.block_frames = pl.block_frames;
    sa.srec = srec; sa.res = st.d_res; sa.loop_start = st.d_loop_start; sa.res_tab = ck.res_tab; sa.sm = sm; sa.rec = pl.rec;
    return FW_LAUNCH(p, 1, 1, launch_sampler(sa, p->stream)) ? FW_PROC_OK : FW_PROC_DEVICE_ERROR;
}

// Biquad or SVF cascade (`filter`) and / or delay line. Two one-channel blocks share a pass as its two row segments: twice the rows
// per launch. The state / ring row of voice v, channel c is v * nc + c; blocks of all nc channels or of one get there with
// srow_mul = nc / C. Every pass of a chunk starts at the same ring cursor, which then advances once.
static int run_temporal(fw_processor* p, const NodeDeviceState* filter, NodeDeviceState* delay, const RowBlock* b, uint32_t nb, uint32_t T, uint32_t zero_first) {
    const uint32_t V = p->num_voices, nc = channels_of(b, nb), D = delay ? delay->params->delay : 0u;
    for (uint32_t i = 0, c = 0; i < nb; i += 2) {
        const uint32_t segs = i + 1 < nb ? 2u : 1u;
        TemporalArgs ta{};
        ta.in = b[i].in; ta.out = b[i].out; ta.in_pitch = (uint32_t)b[i].in_pitch; ta.out_pitch = (uint32_t)b[i].out_pitch;
        ta.R = segs * V * b[i].C; ta.C = b[i].C; ta.T = T; ta.zero_first = zero_first; ta.srow_mul = nc / b[i].C; ta.srow_add = c;
        if (segs == 2) { ta.in2 = b[i + 1].in; ta.out2 = b[i + 1].out; ta.seg_rows = V * b[i].C; }
        if (filter) { ta.svf = filter->kind == FW_NODE_SVF ? 1u : 0u; ta.ns = filter->params->num_stages; ta.coeffs = filter->d_coeffs; ta.state = filter->d_state; }
        if (D) { ta.D = D; ta.ring = delay->d_ring; ta.pos = delay->ring_pos; }
        if (!FW_LAUNCH(p, 3, 1, launch_temporal(ta, p->stream))) return FW_PROC_DEVICE_ERROR;
        c += segs * b[i].C;
    }
    if (D) delay->ring_pos = (uint32_t)(((uint64_t)delay->ring_pos + T) % D);
    return FW_PROC_OK;
}

// ConvReverb: one history + GEMM launch per block; history rows of channel c are c * V .. c * V + V - 1. The history cursor
// advances once per piece, the GEMM's fix-up epoch once per launch. A chunk longer than the history buffers hold
// (kReverbMaxFrames) is processed as consecutive pieces of at most that many frames.
static int run_reverb(fw_processor* p, NodeDeviceState& rs, const RowBlock* b, uint32_t nb, uint32_t T, uint32_t zero_first) {
    const uint32_t V = p->num_voices, H = reverb_hist(rs.params->ir_len);
    for (uint32_t t0 = 0; t0 < T; t0 += NodeDeviceState::kReverbMaxFrames) {
        const uint32_t Tp = std::min(T - t0, NodeDeviceState::kReverbMaxFrames), zf = zero_first > t0 ? std::min(zero_first - t0, Tp) : 0u;
        if (rs.xh_cursor + Tp > rs.xh_pitch || (rs.xh_cursor & 7u)) {  // buffer full (or cursor off the 16-byte TMA grid after an odd-length piece):
            // carry the H most recent samples to the front of the other buffer
            if (!FW_CUDA(cudaMemcpy2DAsync(rs.d_xh[rs.xh_cur ^ 1u], (size_t)rs.xh_pitch * 2, static_cast<const uint16_t*>(rs.d_xh[rs.xh_cur]) + (rs.xh_cursor - H),
                                           (size_t)rs.xh_pitch * 2, (size_t)H * 2, (size_t)V * channels_of(b, nb), cudaMemcpyDeviceToDevice, p->stream))) return FW_PROC_DEVICE_ERROR;
            rs.xh_cur ^= 1u; rs.xh_cursor = H;
        }
        for (uint32_t i = 0, c = 0; i < nb; c += b[i].C, ++i) {
            ReverbCall rc{};
            rc.in = b[i].in + t0; rc.out = b[i].out + t0; rc.in_pitch = (uint32_t)b[i].in_pitch; rc.out_pitch = (uint32_t)b[i].out_pitch; rc.xh = rs.d_xh[rs.xh_cur]; rc.bt = rs.d_bt;
            rc.V = V; rc.C = b[i].C; rc.T = Tp; rc.L = rs.params->ir_len; rc.ir_ch = rs.params->ir_channels; rc.cursor = rs.xh_cursor; rc.pitch = rs.xh_pitch;
            rc.zero_first = zf; rc.chan_base = c;
            rc.ws = rs.d_rv_ws; rc.flags = rs.d_rv_flags; rc.epoch = ++rs.rv_epoch;
            std::string rerr;
            if (!FW_LAUNCH(p, 3, 2, launch_reverb(rc, p->stream, &rerr))) { if (!rerr.empty()) g_dev_err = rerr; return FW_PROC_DEVICE_ERROR; }
        }
        rs.xh_cursor += Tp;
    }
    return FW_PROC_OK;
}

// ---- timed commands (see Cmd in graph.hpp) -------------------------------------------------------------------------------
static NodeDeviceState* state_of(Plan& pl, const NodeParams* node) {
    for (auto& st : pl.states) if (st->params.get() == node) return st.get();
    return nullptr;  // the node is not part of the current schedule: the command is dropped, like a message to a removed processor
}
struct PokeBatch {
    PokeArgs a{}; fw_processor* p; bool ok = true;
    explicit PokeBatch(fw_processor* p_) : p(p_) {}
    void flush() { if (a.n) { ok = ok && FW_CUDA(launch_poke(a, p->stream)); p->launches++; a.n = 0; } }
    void add(void* ptr, uint64_t val, uint8_t bytes, uint32_t count, uint32_t stride) {
        if (a.n == 16) flush();
        a.ptr[a.n] = ptr; a.val[a.n] = val; a.bytes[a.n] = bytes; a.count[a.n] = count; a.stride_bytes[a.n] = stride; ++a.n;
    }
    void f32(float* base, uint32_t voice, uint32_t V, size_t per_voice, size_t off, float v) {  // element `off` of voice's row (or of every voice's)
        uint32_t bits; std::memcpy(&bits, &v, 4);
        if (voice == FW_ALL_VOICES) add(base + off, bits, 4, V, (uint32_t)(per_voice * 4)); else add(base + (size_t)voice * per_voice + off, bits, 4, 1, 0);
    }
};
// apply the commands scheduled at block `b` of this call: parameter stores become ordered device stores, sampler messages are
// staged per node for the control kernel of the chunk that starts here
static bool apply_commands(fw_processor* p, Plan& pl, uint32_t b) {
    const uint32_t V = p->num_voices;
    PokeBatch pk(p);
    for (size_t i = 0; i < p->pend_n; ++i) {
        const Cmd& m = p->pend[i];
        if (m.block != b || m.kind == CMD_SAMPLER) continue;
        NodeDeviceState* st = state_of(pl, m.node);
        if (m.kind == CMD_UPLOAD) {  // ring order: earlier single stores are flushed first, later ones come after this copy
            float* snap = reinterpret_cast<float*>(m.x);
            if (st) {
                float* dst = m.a < 2 ? (m.a < st->n_sm ? st->d_target[m.a] : nullptr) : (coeff_width(st->kind) ? st->d_coeffs : nullptr);
                const size_t cap = m.a < 2 ? (size_t)V : (size_t)V * st->params->num_stages * coeff_width(st->kind);
                pk.flush();
                if (dst && m.y <= cap) pk.ok = pk.ok && FW_CUDA(cudaMemcpyAsync(dst, snap, m.y * sizeof(float), cudaMemcpyHostToDevice, p->stream));  // pageable source: staged before the call returns
            }
            p->ch->to_free.push(snap);  // back to the main thread (never full: one slot per command)
            continue;
        }
        if (!st || (m.voice != FW_ALL_VOICES && m.voice >= V)) continue;
        const uint32_t cnt = m.voice == FW_ALL_VOICES ? V : 1u; const size_t v0 = m.voice == FW_ALL_VOICES ? 0 : m.voice;
        switch (m.kind) {
            case CMD_TARGET: if (m.a < st->n_sm) pk.f32(st->d_target[m.a], m.voice, V, 1, 0, m.f[0]); break;
            case CMD_COEFFS: {
                const uint32_t w = coeff_width(st->kind), ns = st->params->num_stages;
                if (w && m.a < ns) for (uint32_t k = 0; k < w; ++k) pk.f32(st->d_coeffs, m.voice, V, (size_t)ns * w, (size_t)m.a * w + k, m.f[k]);
                break;
            }
            case CMD_RS_SET:
                if (st->kind != FW_NODE_RESAMPLER) break;
                pk.add(st->d_rs_res + v0, m.b, 4, cnt, 4); pk.add(st->d_rs_flags + v0, m.a, 4, cnt, 4); pk.add(st->d_rs_step + v0, m.x, 8, cnt, 8);
                break;
            case CMD_RS_SEEK: if (st->kind == FW_NODE_RESAMPLER) pk.add(st->d_rs_pos + v0, m.x << 32, 8, cnt, 8); break;
            default: break;
        }
    }
    pk.flush();
    if (!pk.ok) return false;
    for (auto& st : pl.samplers) {
        uint32_t n = 0;
        for (size_t i = 0; i < p->pend_n; ++i) { const Cmd& m = p->pend[i]; if (m.block == b && m.kind == CMD_SAMPLER && m.node == st->params.get()) p->cmd_ptrs[n++] = &m; }
        if (!st->stage_sampler(p->cmd_ptrs.data(), n, p->stream)) return false;
    }
    return true;
}

static constexpr uint32_t kGraphEpoch = 0x0fffffffu;  // error-word epoch of replayed chunks: always "current" (see check_device_error)
// One chunk: control kernel + data plane over frames [ck.t0, ck.t0 + ck.Tc) of the caller's rows (ck.Tfull frames long).
static int enqueue_chunk(fw_processor* p, Plan& pl, const float* d_in, float* d_out, const Chunk& ck) {
    const uint32_t V = p->num_voices, T = ck.Tc;
    ++p->call_epoch;
    ControlArgs ca{};
    ca.tables = pl.tables; ca.rec = pl.rec;
    ca.res_tab = ck.res_tab; ca.n_res = ck.n_res;
    for (auto& st : pl.samplers) if (st->cur_n_msgs) ca.smp_msgs = 1;
    if (pl.image.size() <= sizeof(ca.image)) { std::memcpy(ca.image, pl.image.data(), pl.image.size()); ca.image_in_param = 1; }
    ca.flags = pl.d_flags; ca.num_voices = V; ca.frames = T; ca.block_frames = pl.block_frames;
    ca.a = p->sm_a; ca.b = p->sm_b; ca.eps = p->sm_eps; ca.err_value = ((p->capturing ? kGraphEpoch : p->call_epoch) << 4) | 1u;
    if (!FW_LAUNCH(p, 0, 1, launch_control(ca, p->stream))) return FW_PROC_DEVICE_ERROR;

    // ---- data plane: the steps in order (see Plan::Step); the generic lowering's pool buffer reuse is the reference's
    // (compiler.rs:302-412): it is valid for any execution that respects the schedule order, and each step finishes all blocks of the
    // chunk before the next one starts ----
    if (pl.reads_caller_rows && (uint64_t)pl.n_in * ck.Tfull > 0xffffffffull) { g_dev_err = "input rows of more than 2^32 / channels frames"; return FW_PROC_BAD_ARGS; }
    auto out_rows = [&](const Plan::Operand& o) -> float* {
        return o.space == Plan::CALLER_OUT ? d_out + ck.t0 + (size_t)o.index * ck.Tfull : o.space == Plan::POOL ? pl.d_pool + (size_t)o.index * V * T : pl.d_tmp[o.index];
    };
    auto in_rows = [&](const Plan::Operand& o) -> const float* { return o.space == Plan::CALLER_IN ? d_in + ck.t0 + (size_t)o.index * ck.Tfull : out_rows(o); };
    // floats between the channels of one operand, and between its voices: the caller's rows hold n_in / n_out channels per voice
    auto vstride = [&](const Plan::Operand& o) -> uint64_t {
        if (o.space == Plan::POOL || o.space == Plan::SCRATCH) return (uint64_t)o.C * T;
        return (uint64_t)(o.space == Plan::CALLER_IN ? pl.n_in : pl.n_out) * ck.Tfull;
    };
    auto pitch = [&](const Plan::Operand& o) -> uint64_t { return o.space == Plan::POOL || o.space == Plan::SCRATCH ? T : o.C > 1 ? ck.Tfull : vstride(o); };
    RowBlock rows[64];                   // rows[k]: input operand k and output operand k
    const float* in[64]; float* out[64];  // every input and output channel
    for (size_t si = 0; si < pl.steps.size(); ++si) {
        const Plan::Step& sp = pl.steps[si];
        const uint32_t nb = (uint32_t)std::max(sp.in.size(), sp.out.size());
        uint32_t ni = 0, no = 0; uint64_t ivs = 0, ovs = 0;  // channels and voice strides
        uint32_t ni_real = 0;  // in[ni_real..ni) are graph_in ports >= n_in: d_zero (only the fused chain's first stage has them)
        in[0] = in[1] = nullptr; out[0] = out[1] = nullptr;  // chain_args reads prog.c_in slots; the generic bus step has no outputs
        for (uint32_t k = 0; k < nb; ++k) rows[k] = RowBlock{};
        for (uint32_t k = 0; k < sp.in.size(); ++k) {
            const Plan::Operand& o = sp.in[k];
            RowBlock& r = rows[k];
            r.in = in_rows(o); r.in_pitch = pitch(o); r.C = o.C; ivs = vstride(o);
            for (uint32_t c = 0; c < r.C; ++c) {
                const bool zero = o.space == Plan::CALLER_IN && o.index + c >= pl.n_in;
                in[ni++] = zero ? pl.d_zero : r.in + c * r.in_pitch;
                if (!zero) ni_real = ni;
            }
        }
        for (uint32_t k = 0; k < sp.out.size(); ++k) {
            const Plan::Operand& o = sp.out[k];
            RowBlock& r = rows[k];
            r.out = out_rows(o); r.out_pitch = pitch(o); r.C = o.C; ovs = vstride(o);
            for (uint32_t c = 0; c < r.C && (o.space != Plan::CALLER_OUT || o.index + c < pl.n_out); ++c) out[no++] = r.out + c * r.out_pitch;
        }
        // Voice stride of a chain launch from input channel c. Graph_in ports >= n_in (the fused chain's first stage): a second channel is
        // read as +0.0 by the one-channel variant, a launch with no real channel reads the zero row for every voice.
        auto in_stride = [&](ChainProgram& pr, uint32_t c) -> uint64_t {
            if (ni_real == ni) return ivs;
            if (c >= ni_real) return 0;
            if (c + 1 == ni_real && pr.c_in > 1) pr.c_in = 1;
            return ivs;
        };
        const bool caller = !sp.in.empty() && sp.in[0].space == Plan::CALLER_IN;  // Q11 applies to the caller's rows only
        const uint32_t zf = caller ? ck.zero_first : 0u;
        for (uint32_t b : sp.clear) { if (!FW_CUDA(launch_fill(pl.d_pool + (size_t)b * V * T, (size_t)V * T, 0.0f, p->stream))) return FW_PROC_DEVICE_ERROR; p->launches++; }
        int rc = FW_PROC_OK;
        switch (sp.kind) {
            case STEP_SAMPLER: rc = run_sampler(p, pl, ck, *sp.node, pl.smp[sp.sampler_idx].rec, sp.sm0, rows, nb); break;
            case STEP_TEMPORAL: rc = run_temporal(p, sp.node.get(), sp.delay.get(), rows, nb, T, zf); break;
            case STEP_REVERB: rc = run_reverb(p, *sp.node, rows, nb, T, zf); break;
            case STEP_PROG:
                if (pl.bus && si + 1 == pl.steps.size()) {
                    ChainProgram pr = sp.prog;
                    const uint32_t live = pl.bus_width();
                    if (live < pl.c_out) {  // graph_out ports >= n_out do not reach the bus
                        if (live == 0) break;
                        if (pr.c_in > 2) pr.c_in = live;  // graph_out's copy reads only the live channels
                        pr.c_out = std::min(pr.c_out, live);
                    }
                    const uint64_t vs = in_stride(pr, 0);
                    ChainArgs xa = chain_args(pl, ck, pr, in, vs, out, ovs, caller);
                    rc = run_bus_stage(p, pl, xa, live, ck, d_out + ck.t0);
                    break;
                }
                for (uint32_t c = 0, nc = std::min(ni, no); c < (sp.pairs ? nc : 1u); c += 2) {
                    ChainProgram pr = sp.prog;
                    if (sp.pairs && c + 1 == nc) pr.c_in = pr.c_out = 1;
                    pr.c_out = std::min(pr.c_out, no - c);  // graph_out ports >= n_out are not stored
                    if (pr.c_out == 0) continue;
                    const uint64_t vs = in_stride(pr, c);
                    if (!FW_LAUNCH(p, 1, 1, launch_chain(chain_args(pl, ck, pr, in + c, vs, out + c, ovs, caller), false, p->stream))) return FW_PROC_DEVICE_ERROR;
                }
                for (uint32_t c = 0; sp.mask_slot >= 0 && c < no; ++c) {  // test: the inputs output c is made of
                    SilenceFixArgs fa{};
                    fa.out = out[c]; fa.test = sp.prog.c_in == sp.prog.c_out ? 1ull << c : (1ull << sp.prog.c_in) - 1ull;
                    fa.num_voices = V; fa.frames = T; fa.block_frames = pl.block_frames; fa.mask_slot = sp.mask_slot; fa.rec = pl.rec;
                    if (!FW_LAUNCH(p, 1, 1, launch_silence_fix(fa, p->stream))) return FW_PROC_DEVICE_ERROR;
                }
                break;
            case STEP_SUM:
                for (uint32_t c = 0, ports = ni / no; c < no; ++c) {
                    SumArgs sa{};
                    for (uint32_t q = 0; q < ports; ++q) { sa.in[q] = in[q * no + c]; sa.mask_bit[q] = (uint8_t)(q * no + c); }
                    sa.out = out[c]; sa.n_ports = ports; sa.num_voices = V; sa.frames = T; sa.block_frames = pl.block_frames;
                    sa.mask_slot = sp.mask_slot; sa.skip_silent = ports >= 5 ? 1u : 0u;
                    sa.all_mask = ni >= 64 ? ~0ull : (1ull << ni) - 1ull; sa.rec = pl.rec;
                    if (!FW_LAUNCH(p, 1, 1, launch_sum(sa, p->stream))) return FW_PROC_DEVICE_ERROR;
                }
                break;
            case STEP_RESAMPLER: {
                NodeDeviceState& st = *sp.node;
                ResamplerArgs ra{};
                for (uint32_t c = 0; c < no; ++c) ra.out[c] = out[c];
                ra.out_vstride = ovs; ra.n_out = no; ra.num_voices = V; ra.frames = T; ra.taps = st.params->rs_taps;
                uint32_t lg = 0; while ((1u << lg) < st.params->rs_phases) ++lg;
                ra.phase_shift = 32 - lg;
                ra.table = st.d_rs_table; ra.pos = st.d_rs_pos; ra.step = st.d_rs_step; ra.flags = st.d_rs_flags; ra.res = st.d_rs_res; ra.res_tab = ck.res_tab;
                if (!FW_LAUNCH(p, 3, 2, launch_resampler(ra, st.d_rs_pos, p->stream))) return FW_PROC_DEVICE_ERROR;
                break;
            }
            case STEP_CUSTOM: {  // AudioNodeProcessor::process for all voices and blocks at once (fw_node_vtable::process_device)
                NodeDeviceState& st = *sp.node;
                const uint32_t nblk = (T + pl.block_frames - 1) / pl.block_frames;
                uint64_t* masks = pl.d_custom_masks[sp.custom_idx];
                if (!FW_CUDA(launch_expand_masks(pl.rec, (uint32_t)sp.mask_slot, V, nblk, masks, p->stream))) return FW_PROC_DEVICE_ERROR;
                p->launches++;
                fw_device_block blk{};
                blk.num_voices = V; blk.num_inputs = ni; blk.num_outputs = no; blk.block_frames = pl.block_frames; blk.num_blocks = nblk;
                blk.stream_status = p->cur_stream_status; blk.frames = T; blk.in_voice_stride = T; blk.out_voice_stride = T; blk.inputs = in; blk.outputs = out;
                blk.in_silence_masks = masks; blk.stream_time_secs = p->cur_stream_time; blk.cuda_stream = p->stream; blk.user_cx = p->user_cx;
                ProfScope ps(p, 1);
                if (st.params->custom->vt.process_device(st.custom_proc, &blk) != 0) { g_dev_err = std::string("custom node '") + st.params->custom->debug_name + "': process_device failed"; return FW_PROC_DEVICE_ERROR; }
                break;
            }
        }
        if (rc != FW_PROC_OK) return rc;
    }
    if (pl.n_out > pl.c_out) {  // caller output rows >= c_out, per voice or on the bus, are +0.0 (util.rs:96)
        const uint32_t groups = pl.bus ? 1u : V;
        if (!FW_LAUNCH(p, 1, 1, launch_zero_rows(d_out + ck.t0 + (size_t)pl.c_out * ck.Tfull, T, ck.Tfull, pl.n_out - pl.c_out, groups, (uint64_t)pl.n_out * ck.Tfull, p->stream))) return FW_PROC_DEVICE_ERROR;
    }
    return FW_PROC_OK;
}

// A steady chunk — same plan, same buffers, same frames, no command or upload at its start — is the same launch sequence with the
// same arguments every time: it is captured into a CUDA graph the second time it is seen and replayed from then on (one
// cudaGraphLaunch instead of one launch per kernel; what counts for block-sized calls, where the host's launch cost exceeds the
// kernels' run time). Programmatic-dependent-launch edges are kept by the capture.
static int run_chunk(fw_processor* p, Plan& pl, const float* d_in, float* d_out, const Chunk& ck, bool steady) {
    if (!steady || !pl.graphable || p->graphs_off || p->profiling || p->world > 1 || ck.zero_first) return enqueue_chunk(p, pl, d_in, d_out, ck);
    fw_processor::GraphEntry* e = nullptr; fw_processor::GraphEntry* lru = &p->graphs[0];
    for (auto& g : p->graphs) {
        if (g.plan == &pl && g.d_in == d_in && g.d_out == d_out && g.t0 == ck.t0 && g.Tc == ck.Tc && g.Tfull == ck.Tfull && g.res_tab == ck.res_tab && g.n_res == ck.n_res) { e = &g; break; }
        if (g.stamp < lru->stamp) lru = &g;
    }
    if (!e) {  // first sight: remember the key, run normally
        e = lru;
        if (e->exec) { cudaGraphExecDestroy(e->exec); e->exec = nullptr; }
        e->plan = &pl; e->d_in = d_in; e->d_out = d_out; e->t0 = ck.t0; e->Tc = ck.Tc; e->Tfull = ck.Tfull; e->res_tab = ck.res_tab; e->n_res = ck.n_res; e->seen = 0;
    }
    e->stamp = ++p->graph_stamp;
    if (e->exec) {
        if (!FW_CUDA(cudaGraphLaunch(e->exec, p->stream))) return FW_PROC_DEVICE_ERROR;
        ++p->graph_replays; p->launches += e->seen;  // `seen` holds the kernel count of the captured sequence once instantiated
        return FW_PROC_OK;
    }
    if (++e->seen < 2) return enqueue_chunk(p, pl, d_in, d_out, ck);
    // second sight: capture, instantiate, launch
    const uint64_t l0 = p->launches;
    if (cudaStreamBeginCapture(p->stream, cudaStreamCaptureModeThreadLocal) != cudaSuccess) { cudaGetLastError(); p->graphs_off = true; return enqueue_chunk(p, pl, d_in, d_out, ck); }
    p->capturing = true;
    const int rc = enqueue_chunk(p, pl, d_in, d_out, ck);
    p->capturing = false;
    cudaGraph_t graph = nullptr;
    const cudaError_t ce = cudaStreamEndCapture(p->stream, &graph);
    const uint32_t n_launch = (uint32_t)(p->launches - l0);
    p->launches = l0;
    if (rc != FW_PROC_OK || ce != cudaSuccess || !graph || cudaGraphInstantiate(&e->exec, graph, 0) != cudaSuccess) {
        cudaGetLastError();
        if (graph) cudaGraphDestroy(graph);
        e->exec = nullptr; e->plan = nullptr; p->graphs_off = true;  // capture is not available here: stay on plain launches
        return enqueue_chunk(p, pl, d_in, d_out, ck);
    }
    cudaGraphDestroy(graph);
    e->seen = n_launch;
    if (!FW_CUDA(cudaGraphLaunch(e->exec, p->stream))) return FW_PROC_DEVICE_ERROR;
    ++p->graph_replays; p->launches += n_launch;
    return FW_PROC_OK;
}

// One process_* call on device buffers: d_in [V][c_in][T]; d_out [V][c_out][T] or bus [c_out][T]. The call is processed as
// consecutive chunks; a chunk boundary is (a) every plan.chunk_frames frames — the stretch device memory was reserved for —
// and (b) every block at which a timed command takes effect. Messages from the context (new schedule, Stop; processor.rs:
// 167-206) are polled at every chunk boundary, i.e. per block whenever the host asks for per-block control.
static int proc_call(fw_processor* p, const float* d_in, float* d_out, uint32_t n_in, uint32_t n_out, uint64_t frames64) {
    if (frames64 > 0x7fffffffull) return FW_PROC_BAD_ARGS;
    const uint32_t T = (uint32_t)frames64, V = p->num_voices;
    if (n_in != p->n_in || n_out != p->n_out) { g_dev_err = "channel counts do not match the activated stream"; return FW_PROC_BAD_ARGS; }
    const size_t out_rows = (size_t)(p->bus ? 1 : V) * n_out;
    cudaSetDevice(p->device);
    // zero frames [t0, T) of every output row
    auto silence_from = [&](uint32_t t0) {
        if (!out_rows || t0 >= T) return;
        if (t0 == 0) launch_fill(d_out, out_rows * T, 0.0f, p->stream);
        else cudaMemset2DAsync(d_out + t0, (size_t)T * 4, 0, (size_t)(T - t0) * 4, out_rows, p->stream);
        p->launches++;
    };
    if (!p->running) { silence_from(0); return FW_PROC_DROP_PROCESSOR; }                   // processor.rs:71-74
    if (!p->plan) { proc_poll(p); p->pending_zero_first = false; if (!p->running) { silence_from(0); return FW_PROC_DROP_PROCESSOR; } }  // :76-84
    if (!p->plan || T == 0) { silence_from(0); return FW_PROC_OK; }                        // :86-89
    // drain the command ring (sampler.rs:331 / volume.rs:92 happen at block granularity below)
    {
        Cmd m;
        bool any = false;
        while (p->pend_n < p->pend.size() && p->ch->cmds.pop(&m)) { p->pend[p->pend_n++] = m; any = true; }
        if (any) {
            p->ch->drain_epoch.fetch_add(1, std::memory_order_release);
            for (size_t i = 1; i < p->pend_n; ++i) {  // stable insertion sort by block: push order is almost always sorted already
                if (p->pend[i].block >= p->pend[i - 1].block) continue;
                Cmd key = p->pend[i]; size_t j = i;
                while (j > 0 && p->pend[j - 1].block > key.block) { p->pend[j] = p->pend[j - 1]; --j; }
                p->pend[j] = key;
            }
        }
    }
    const uint32_t F = p->max_block_frames, n_blocks = (T + F - 1) / F;
    uint32_t b = 0; size_t next_cmd = 0;  // pend[next_cmd..) have block >= b
    int rc = FW_PROC_OK;
    while (b < n_blocks) {
        proc_poll(p);                                                                        // process_block :214
        if (!p->running) { silence_from(b * F); rc = FW_PROC_DROP_PROCESSOR; break; }        // :150-155
        Plan& pl = *p->plan;
        while (next_cmd < p->pend_n && p->pend[next_cmd].block < b) ++next_cmd;
        const bool have_cmds = next_cmd < p->pend_n && p->pend[next_cmd].block == b;
        if (have_cmds || !pl.samplers.empty()) { if (!apply_commands(p, pl, b)) return FW_PROC_DEVICE_ERROR; }
        size_t nc = next_cmd; while (nc < p->pend_n && p->pend[nc].block == b) ++nc;
        uint32_t b_end = std::min(n_blocks, b + pl.chunk_blocks);
        if (nc < p->pend_n && p->pend[nc].block < b_end) b_end = p->pend[nc].block;          // the next timed command splits the call
        next_cmd = nc;
        Chunk ck{b * F, std::min(T, b_end * F) - b * F, T, 0, nullptr, 0};
        // one snapshot of the resource table for every sampler and resampler of the chunk; it holds every handle they use (the main
        // thread checks a handle against the table before it sends it, and the table only grows)
        if (pl.res) pl.res->snapshot(&ck.res_tab, &ck.n_res);
        if (p->pending_zero_first) { ck.zero_first = std::min(pl.block_frames, ck.Tc); p->pending_zero_first = false; }  // Q11
        bool steady = true;  // no sampler message rides in this chunk's control arguments (stores and uploads precede the chunk: they do not change it)
        for (auto& st : pl.samplers) if (st->cur_n_msgs) steady = false;
        const int erc = run_chunk(p, pl, d_in, d_out, ck, steady);
        if (erc != FW_PROC_OK) return erc;
        b = b_end;
    }
    // commands beyond this call stay queued, their block offsets re-based to the next call
    size_t keep = 0;
    for (size_t i = 0; i < p->pend_n; ++i) if (p->pend[i].block >= n_blocks) { Cmd m = p->pend[i]; m.block -= n_blocks; p->pend[keep++] = m; }
    p->pend_n = keep;
    return rc;
}

// The graph_out mask covers the stream's n_out channels (schedule.rs:269); channels >= graph_out's ports are never flagged, so with
// more than one voice a bus with such channels is never all silent (the tree's SumNodes, sum.rs:52-56).
static uint64_t bus_mask_from(const uint64_t* masks, uint32_t V, uint32_t n_out) {
    const uint64_t all = n_out >= 64 ? ~0ull : ((1ull << n_out) - 1ull);
    if (V == 1) return masks[0] & all;
    for (uint32_t v = 0; v < V; ++v) if ((masks[v] & all) != all) return 0;
    return all;
}

int fw_processor_process_planar_device(fw_processor* p, const float* d_in, float* d_out, uint32_t n_in, uint32_t n_out, uint64_t frames, double stream_time_secs, uint32_t stream_status) {
    if (!p) return FW_PROC_BAD_ARGS;
    p->cur_stream_time = stream_time_secs; p->cur_stream_status = stream_status;
    return proc_call(p, d_in, d_out, n_in, n_out, frames);
}

// error word of the plan: (chunk epoch << 4) | code, written by the control kernel (1: record budget) or the exchange (2: peer time-out);
// an error counts when it comes from a chunk of epoch since_epoch or later
static int check_device_error(fw_processor* p, uint32_t since_epoch) {
    if (!p->plan) return 0;
    const uint32_t e = *p->h_err;
    if ((e & 15u) == 0 || ((e >> 4) != kGraphEpoch && (int32_t)((e >> 4) - (since_epoch & 0x0fffffffu)) < 0)) return 0;
    if ((e >> 4) == kGraphEpoch) cudaMemsetAsync(p->plan->rec.error, 0, 4, p->stream);  // a replayed chunk cannot stamp its epoch: report once, then clear
    g_dev_err = (e & 15u) == 2 ? "master-bus exchange timed out waiting for a peer rank" : "control pass overflowed its transient-block budget (a gain jump beyond 10000 %?)";
    publish_error();
    return FW_PROC_DEVICE_ERROR;
}

// One call on host buffers, in host chunks of at most max_call_frames (the staging buffers were sized for that at activate): per host
// chunk, stage_in(t0, Tc) puts the caller's frames [t0, t0 + Tc) into d_in, proc_call runs them and stage_out(t0, Tc, rc) returns
// d_out to the caller. After a drop, zero_rest(t0) zeroes the caller's output from frame t0 on. One synchronise at the end, then the
// error word is checked for every chunk of the call and the graph_out silence mask goes to out_mask (when not null).
extern "C++" {  // a template inside the C ABI block
template <class StageIn, class StageOut, class ZeroRest>
static int host_call(fw_processor* p, uint32_t n_in, uint32_t n_out, uint64_t frames, double stream_time_secs, uint32_t stream_status, uint64_t* out_mask,
                     StageIn&& stage_in, StageOut&& stage_out, ZeroRest&& zero_rest) {
    p->cur_stream_time = stream_time_secs; p->cur_stream_status = stream_status;
    cudaSetDevice(p->device);
    if (n_in != p->n_in || n_out != p->n_out) { g_dev_err = "channel counts do not match the activated stream"; return FW_PROC_BAD_ARGS; }
    const uint32_t V = p->num_voices, since_epoch = p->call_epoch + 1;
    int rc = FW_PROC_OK;
    uint64_t t0 = 0;
    do {
        const uint64_t Tc = std::min<uint64_t>(frames - t0, p->max_call_frames);
        if (!stage_in(t0, Tc)) return FW_PROC_DEVICE_ERROR;
        rc = proc_call(p, p->d_in, p->d_out, n_in, n_out, Tc);
        if (rc < 0) return rc;
        join_side(p);
        if (!stage_out(t0, Tc, rc)) return FW_PROC_DEVICE_ERROR;
        t0 += Tc;
    } while (t0 < frames && rc == FW_PROC_OK);
    if (rc == FW_PROC_DROP_PROCESSOR && t0 < frames) zero_rest(t0);
    const bool ran = rc == FW_PROC_OK && p->plan && frames > 0;
    if (ran) {
        if (out_mask) cudaMemcpyAsync(p->h_masks, p->plan->rec.gout_mask, sizeof(uint64_t) * V, cudaMemcpyDeviceToHost, p->stream);
        cudaMemcpyAsync(p->h_err, p->plan->rec.error, sizeof(uint32_t), cudaMemcpyDeviceToHost, p->stream);
    }
    if (!FW_CUDA(cudaStreamSynchronize(p->stream))) return FW_PROC_DEVICE_ERROR;
    if (ran) {
        if (check_device_error(p, since_epoch)) return FW_PROC_DEVICE_ERROR;
        if (out_mask) *out_mask = p->bus ? bus_mask_from(p->h_masks, V, n_out) : p->h_masks[0] & (n_out >= 64 ? ~0ull : (1ull << n_out) - 1ull);
    }
    return rc;
}
}  // extern "C++"

int fw_processor_process_planar(fw_processor* p, const float* in, float* out, uint32_t n_in, uint32_t n_out, uint64_t frames, double stream_time_secs, uint32_t stream_status, uint64_t* out_mask) {
    if (!p) return FW_PROC_BAD_ARGS;
    if (out_mask) *out_mask = 0;
    const size_t in_rows = (size_t)p->num_voices * n_in, out_rows = (size_t)(p->bus ? 1 : p->num_voices) * n_out;
    return host_call(p, n_in, n_out, frames, stream_time_secs, stream_status, out_mask,
        [&](uint64_t t0, uint64_t Tc) { return !in_rows || !Tc || FW_CUDA(cudaMemcpy2DAsync(p->d_in, Tc * 4, in + t0, frames * 4, Tc * 4, in_rows, cudaMemcpyHostToDevice, p->stream)); },
        [&](uint64_t t0, uint64_t Tc, int) { return !out_rows || !Tc || FW_CUDA(cudaMemcpy2DAsync(out + t0, frames * 4, p->d_out, Tc * 4, Tc * 4, out_rows, cudaMemcpyDeviceToHost, p->stream)); },
        [&](uint64_t t0) { for (size_t r = 0; r < out_rows; ++r) std::memset(out + r * frames + t0, 0, (frames - t0) * 4); });
}

int fw_processor_process_interleaved(fw_processor* p, const float* in, float* out, uint32_t n_in, uint32_t n_out, uint64_t frames, double stream_time_secs, uint32_t stream_status) {
    if (!p) return FW_PROC_BAD_ARGS;
    const uint32_t V = p->num_voices, Vo = p->bus ? 1 : V;
    return host_call(p, n_in, n_out, frames, stream_time_secs, stream_status, nullptr,
        [&](uint64_t t0, uint64_t Tc) {  // voice v's frames [t0, t0 + Tc) are one contiguous run of Tc * n_in floats
            if (!n_in || !Tc) return true;
            if (!FW_CUDA(cudaMemcpy2DAsync(p->d_inter, Tc * n_in * 4, in + t0 * n_in, frames * n_in * 4, Tc * n_in * 4, V, cudaMemcpyHostToDevice, p->stream))) return false;
            if (!FW_CUDA(launch_deinterleave(p->d_inter, p->d_in, V, n_in, (uint32_t)Tc, p->stream))) return false;
            p->launches++;
            return true;
        },
        [&](uint64_t t0, uint64_t Tc, int rc) {
            if (!n_out || !Tc) return true;
            const uint64_t* masks = nullptr;
            if (rc == FW_PROC_OK && p->plan) {
                if (p->bus) { launch_bus_mask(p->plan->rec.gout_mask, V, n_out, p->plan->d_bus_mask, p->stream); p->launches++; masks = p->plan->d_bus_mask; }
                else masks = p->plan->rec.gout_mask;
            }
            if (!FW_CUDA(launch_interleave(p->d_out, p->d_inter, masks, Vo, n_out, (uint32_t)Tc, p->max_block_frames, p->stream))) return false;
            p->launches++;
            return FW_CUDA(cudaMemcpy2DAsync(out + t0 * n_out, frames * n_out * 4, p->d_inter, Tc * n_out * 4, Tc * n_out * 4, Vo, cudaMemcpyDeviceToHost, p->stream));
        },
        [&](uint64_t t0) { for (size_t v = 0; v < Vo; ++v) std::memset(out + (v * frames + t0) * n_out, 0, (frames - t0) * n_out * 4); });
}

void fw_processor_free(fw_processor* p) {  // Drop processor.rs:251-263
    if (!p) return;
    cudaSetDevice(p->device);
    join_side(p);
    cudaStreamSynchronize(p->stream);
    if (p->side) cudaStreamSynchronize(p->side);
    ProcToCtx m; m.kind = 1; m.plan = p->plan; m.user_cx = p->user_cx;
    if (!p->ch->to_ctx.push(m)) delete p->plan;
    for (size_t i = 0; i < p->pend_n; ++i) if (p->pend[i].kind == CMD_UPLOAD) delete[] reinterpret_cast<float*>(p->pend[i].x);
    delete p;
}

// ---- device plumbing ----------------------------------------------------------------------------
int fw_device_count(void) { int n = 0; if (!FW_CUDA(cudaGetDeviceCount(&n))) return 0; return n; }
const char* fw_last_device_error(void) {
    if (!g_dev_err.empty()) return g_dev_err.c_str();
    static thread_local std::string copy;
    { std::lock_guard<std::mutex> lk(g_err_mu); copy = g_err_any; }
    return copy.c_str();
}
void* fw_dev_malloc(int device, uint64_t bytes) { void* p = nullptr; if (!FW_CUDA(cudaSetDevice(device)) || !FW_CUDA(cudaMalloc(&p, bytes))) return nullptr; return p; }
void fw_dev_free(int device, void* p) { cudaSetDevice(device); cudaFree(p); }
void* fw_host_alloc_pinned(uint64_t bytes) { void* p = nullptr; if (!FW_CUDA(cudaMallocHost(&p, bytes))) return nullptr; return p; }
void fw_host_free_pinned(void* p) { cudaFreeHost(p); }
int fw_processor_h2d(fw_processor* p, void* dst, const void* src, uint64_t bytes) { cudaSetDevice(p->device); return FW_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, p->stream)) ? 0 : -1; }
int fw_processor_d2h(fw_processor* p, void* dst, const void* src, uint64_t bytes) { cudaSetDevice(p->device); join_side(p); return FW_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, p->stream)) ? 0 : -1; }
int fw_processor_sync(fw_processor* p) {
    cudaSetDevice(p->device);
    join_side(p);
    if (!FW_CUDA(cudaStreamSynchronize(p->stream))) return -1;
    if (p->plan) { cudaMemcpy(p->h_err, p->plan->rec.error, 4, cudaMemcpyDeviceToHost); const uint32_t since = p->synced_epoch + 1; p->synced_epoch = p->call_epoch; if (check_device_error(p, since)) return -1; }
    return 0;
}
int fw_processor_event_record(fw_processor* p, int slot) { if (slot < 0 || slot > 3) return -1; cudaSetDevice(p->device); join_side(p); return FW_CUDA(cudaEventRecord(p->ev[slot], p->stream)) ? 0 : -1; }
float fw_processor_event_elapsed_ms(fw_processor* p, int a, int b) {
    float ms = -1.0f; cudaSetDevice(p->device);
    if (!FW_CUDA(cudaEventSynchronize(p->ev[b])) || !FW_CUDA(cudaEventElapsedTime(&ms, p->ev[a], p->ev[b]))) return -1.0f;
    return ms;
}
uint64_t fw_processor_kernel_launches(fw_processor* p) { return p->launches; }
uint64_t fw_processor_graph_replays(fw_processor* p) { return p->graph_replays; }
int fw_processor_profile(fw_processor* p, int enable) {
    cudaSetDevice(p->device);
    if (enable && p->prof_ev.empty()) {
        p->prof_ev.resize(2 * 4096); p->prof_class.assign(4096, 0);
        for (auto& e : p->prof_ev) if (!FW_CUDA(cudaEventCreate(&e))) return -1;
    }
    p->profiling = enable != 0; p->prof_used = 0;
    return 0;
}
int fw_processor_profile_read(fw_processor* p, double* ms4, uint64_t* n4) {
    cudaSetDevice(p->device);
    if (!FW_CUDA(cudaStreamSynchronize(p->stream))) return -1;
    for (int i = 0; i < 4; ++i) { ms4[i] = 0.0; n4[i] = 0; }
    for (size_t i = 0; i + 1 < p->prof_used; i += 2) {
        float ms = 0.0f;
        if (!FW_CUDA(cudaEventElapsedTime(&ms, p->prof_ev[i], p->prof_ev[i + 1]))) return -1;
        const int cls = p->prof_class[i / 2] & 3;
        ms4[cls] += ms; n4[cls] += 1;
    }
    p->prof_used = 0;
    return 0;
}
int fw_processor_l2_flush(fw_processor* p) {
    cudaSetDevice(p->device);
    const size_t n = (size_t)64 << 20;  // 256 MiB of f32 > 50 MB L2
    if (!p->d_flush && !(p->d_flush = p->mem.dev<float>(n, false))) return -1;
    if (!FW_CUDA(launch_fill(p->d_flush, n, 1.0f, p->stream))) return -1;
    return 0;
}
// ---- pull-style stream backend (SURVEY f3) -------------------------------------------------------
struct fw_stream {
    fw_processor* p = nullptr; uint32_t n_out = 0, period = 0, n_periods = 0, sample_rate = 0;
    std::vector<float> ring;                                    // [n_periods][period][n_out]
    std::atomic<uint64_t> produced{0}, consumed{0};             // periods
    std::atomic<uint32_t> pending_status{0};                    // flags for the next rendered period (OUTPUT_UNDERFLOW)
    std::atomic<bool> stop{false}, dropped{false};
    uint64_t cursor = 0, frames_delivered = 0;                  // consumer side
    std::mutex mu; std::condition_variable cv; std::thread th;
};
static void stream_producer(fw_stream* s) {
    uint64_t frames_rendered = 0;
    while (!s->stop.load(std::memory_order_acquire)) {
        const uint64_t prod = s->produced.load(std::memory_order_relaxed);
        if (prod - s->consumed.load(std::memory_order_acquire) >= s->n_periods) {  // ring full: sleep until the consumer frees a period
            std::unique_lock<std::mutex> lk(s->mu);
            s->cv.wait_for(lk, std::chrono::milliseconds(1));
            continue;
        }
        float* dst = s->ring.data() + (size_t)(prod % s->n_periods) * s->period * s->n_out;
        const uint32_t status = s->pending_status.exchange(0, std::memory_order_acq_rel);
        const int rc = fw_processor_process_interleaved(s->p, nullptr, dst, 0, s->n_out, s->period, (double)frames_rendered / (double)s->sample_rate, status);
        if (rc != FW_PROC_OK) {  // DropProcessor (lib.rs:440-448) or a device error: this period is silence, and so is everything after it
            if (rc < 0) { std::fill(dst, dst + (size_t)s->period * s->n_out, 0.0f); publish_error(); }  // visible to fw_last_device_error() on the consumer's thread
            s->dropped.store(true, std::memory_order_release);
            s->produced.store(prod + 1, std::memory_order_release);
            return;
        }
        frames_rendered += s->period;
        s->produced.store(prod + 1, std::memory_order_release);
    }
}
fw_stream* fw_stream_open(fw_processor* p, uint32_t n_out, uint32_t sample_rate, uint32_t period_frames, uint32_t ring_periods) {
    if (!p || n_out == 0 || n_out > 64 || sample_rate == 0 || period_frames == 0 || ring_periods < 2) { g_dev_err = "bad stream arguments"; return nullptr; }
    if (!p->bus && p->num_voices != 1) { g_dev_err = "a stream needs one output: num_voices == 1 or master_bus == 1"; return nullptr; }
    auto* s = new fw_stream();
    s->p = p; s->n_out = n_out; s->period = period_frames; s->n_periods = ring_periods; s->sample_rate = sample_rate;
    s->ring.assign((size_t)ring_periods * period_frames * n_out, 0.0f);
    s->th = std::thread(stream_producer, s);
    return s;
}
int64_t fw_stream_pull(fw_stream* s, float* out, uint64_t frames, uint32_t* status, double* stream_time_secs) {
    if (!s || (!out && frames)) return -1;
    if (status) *status = 0;
    if (stream_time_secs) *stream_time_secs = (double)s->frames_delivered / (double)s->sample_rate;
    uint64_t done = 0;
    while (done < frames) {
        const uint64_t cons = s->consumed.load(std::memory_order_relaxed);
        if (cons == s->produced.load(std::memory_order_acquire)) {
            if (s->dropped.load(std::memory_order_acquire)) {  // no processor any more: silence, not an underflow
                std::fill(out + done * s->n_out, out + frames * s->n_out, 0.0f);
                s->frames_delivered += frames - done;
                return (int64_t)frames;
            }
            std::fill(out + done * s->n_out, out + frames * s->n_out, 0.0f);  // underflow: the consumer outran the producer
            s->pending_status.fetch_or(FW_STREAM_OUTPUT_UNDERFLOW, std::memory_order_acq_rel);
            if (status) *status |= FW_STREAM_OUTPUT_UNDERFLOW;
            break;
        }
        const uint64_t n = std::min<uint64_t>(s->period - s->cursor, frames - done);
        const float* src = s->ring.data() + ((size_t)(cons % s->n_periods) * s->period + s->cursor) * s->n_out;
        std::memcpy(out + done * s->n_out, src, (size_t)n * s->n_out * sizeof(float));
        done += n; s->cursor += n;
        if (s->cursor == s->period) { s->cursor = 0; s->consumed.store(cons + 1, std::memory_order_release); s->cv.notify_one(); }
    }
    s->frames_delivered += done;
    return (int64_t)done;
}
uint64_t fw_stream_frames_ready(fw_stream* s) {
    if (!s) return 0;
    const uint64_t periods = s->produced.load(std::memory_order_acquire) - s->consumed.load(std::memory_order_relaxed);
    return periods * s->period - (periods ? s->cursor : 0);
}
void fw_stream_close(fw_stream* s) {
    if (!s) return;
    s->stop.store(true, std::memory_order_release);
    s->cv.notify_all();
    if (s->th.joinable()) s->th.join();
    delete s;
}

int fw_comm_unique_id(uint8_t* id128) {
    if (!id128 || !g_nccl.load()) return -1;
    NcclUniqueId id;
    if (!g_nccl.ok(g_nccl.GetUniqueId(&id), "ncclGetUniqueId")) return -1;
    std::memcpy(id128, id.internal, 128);
    return 0;
}
int fw_processor_comm_init(fw_processor* p, int rank, int world, const uint8_t* id128) {
    if (!p || !id128 || world < 1 || world > 16 || rank < 0 || rank >= world) { g_dev_err = "bad comm arguments (1 <= world <= 16)"; return -1; }
    if (world == 1) { p->rank = 0; p->world = 1; return 0; }
    if (!g_nccl.load()) return -1;
    cudaSetDevice(p->device);
    NcclUniqueId id; std::memcpy(id.internal, id128, 128);
    if (!g_nccl.ok(g_nccl.CommInitRank(&p->nccl_comm, world, id, rank), "ncclCommInitRank")) return -1;
    int prio_lo = 0, prio_hi = 0;
    cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi);  // the exchange must not queue behind the next call's chain CTAs
    if (!FW_CUDA(cudaStreamCreateWithPriority(&p->side, cudaStreamNonBlocking, prio_hi)) || !FW_CUDA(cudaEventCreateWithFlags(&p->ev_exchange_done[0], cudaEventDisableTiming)) ||
        !FW_CUDA(cudaEventCreateWithFlags(&p->ev_exchange_done[1], cudaEventDisableTiming))) return -1;
    p->rank = rank; p->world = world;
    for (int q = 0; q < 2; ++q) {
        p->d_bus_local[q] = p->mem.dev<float>((size_t)p->n_out * p->max_call_frames, false); p->d_gather[q] = p->mem.dev<float>((size_t)world * p->n_out * p->max_call_frames, false);
    }
    p->d_handover = p->mem.dev<uint32_t>(2);  // [0] epoch word, [1] last-CTA counter of the signalling combine
    return p->mem.ok() ? 0 : -1;
}
// Host-buffer all-gather over the processor's communicator: what a torch-free driver needs for barriers, max-over-ranks
// timing and result cross-checks (bench.py, tests/multigpu_worker.py). Not on the audio path.
int fw_processor_comm_allgather(fw_processor* p, const void* send, void* recv, uint64_t bytes) {
    if (!p || !send || !recv || bytes == 0) return -1;
    if (p->world == 1) { std::memcpy(recv, send, bytes); return 0; }
    if (!p->nccl_comm) { g_dev_err = "comm_allgather: no communicator (call processor_comm_init first)"; return -1; }
    cudaSetDevice(p->device);
    uint8_t* d = nullptr;
    if (!FW_CUDA(cudaMalloc(&d, bytes * (size_t)p->world))) return -1;
    bool ok = FW_CUDA(cudaMemcpyAsync(d + bytes * (size_t)p->rank, send, bytes, cudaMemcpyHostToDevice, p->side)) &&
              g_nccl.ok(g_nccl.AllGather(d + bytes * (size_t)p->rank, d, bytes, /*ncclInt8*/ 0, p->nccl_comm, p->side), "ncclAllGather(host)") &&
              FW_CUDA(cudaMemcpyAsync(recv, d, bytes * (size_t)p->world, cudaMemcpyDeviceToHost, p->side)) && FW_CUDA(cudaStreamSynchronize(p->side));
    cudaFree(d);
    return ok ? 0 : -1;
}

}  // extern "C"
