// graph.hpp — product host side: AudioGraph + schedule compiler (pure C++, no CUDA).
//
// Mirrors the observable behaviour of firewheel-graph's control plane so the C ABI is a
// drop-in: crates/firewheel-graph/src/graph.rs (AudioGraph), graph/compiler.rs (Kahn sort
// + buffer assignment) and graph/error.rs. Node / edge ids are generational slot indices
// with thunderdome 0.6.1's observable rules (LIFO slot reuse, generation bump on reuse,
// ascending-slot iteration) because ids cross the boundary.
//
// Internals are NOT the reference's: slots live in flat vectors with an explicit free
// stack, adjacency is rebuilt into CSR-style per-node port tables, and buffer lifetimes
// are tracked with plain reference counts. The compiled result additionally carries what
// the device lowering needs (per-port producer links).
#pragma once
#include <atomic>
#include <cstdint>
#include <cstring>
#include <deque>
#include <memory>
#include <mutex>
#include <string>
#include <unordered_map>
#include <unordered_set>
#include <vector>

#include "../../include/fw_b200.h"
#include "plan.hpp"

namespace fw {

struct Id {
    uint32_t slot = UINT32_MAX, gen = UINT32_MAX;
    bool operator==(const Id& o) const { return slot == o.slot && gen == o.gen; }
    bool operator!=(const Id& o) const { return !(*this == o); }
    uint64_t pack() const { return (uint64_t)slot | ((uint64_t)gen << 32); }
    static Id unpack(uint64_t v) { return Id{(uint32_t)(v & 0xffffffffu), (uint32_t)(v >> 32)}; }
};

// Generational slot table. Free slots are reused most-recently-freed first.
template <class T>
class SlotTable {
    struct Slot { uint32_t gen = 0; bool live = false; T value{}; };
    std::vector<Slot> slots_;
    std::vector<uint32_t> free_;  // stack
    uint32_t live_ = 0;

  public:
    Id insert(T v) {
        uint32_t s;
        if (!free_.empty()) { s = free_.back(); free_.pop_back(); }
        else { s = (uint32_t)slots_.size(); slots_.emplace_back(); }
        Slot& sl = slots_[s];
        sl.gen += 1; sl.live = true; sl.value = std::move(v);
        ++live_;
        return Id{s, sl.gen};
    }
    bool erase(Id id, T* out = nullptr) {
        if (!has(id)) return false;
        Slot& sl = slots_[id.slot];
        if (out) *out = std::move(sl.value);
        sl.value = T{}; sl.live = false;
        free_.push_back(id.slot);
        --live_;
        return true;
    }
    bool has(Id id) const { return id.slot < slots_.size() && slots_[id.slot].live && slots_[id.slot].gen == id.gen; }
    T* find(Id id) { return has(id) ? &slots_[id.slot].value : nullptr; }
    const T* find(Id id) const { return has(id) ? &slots_[id.slot].value : nullptr; }
    T* by_slot(uint32_t s, Id* id = nullptr) {
        if (s >= slots_.size() || !slots_[s].live) return nullptr;
        if (id) *id = Id{s, slots_[s].gen};
        return &slots_[s].value;
    }
    uint32_t size() const { return live_; }
    uint32_t slot_count() const { return (uint32_t)slots_.size(); }
    template <class F> void each(F&& f) {
        for (uint32_t s = 0; s < slots_.size(); ++s) if (slots_[s].live) f(Id{s, slots_[s].gen}, slots_[s].value);
    }
};

// A user node behind the plugin vtable (include/fw_b200.h fw_node_vtable): the graph's `Box<dyn AudioNode>`.
struct CustomNode {
    fw_node_vtable vt{}; void* node = nullptr; fw_audio_node_info info{}; std::string debug_name;
    ~CustomNode() { if (vt.drop_node) vt.drop_node(node); }
};

// ---- main thread -> stream side commands (wait-free SPSC ring, see Channels in runtime.cu) ----------------------------
// The reference's per-node message rings (sampler.rs:14,205-208) and relaxed-atomic parameter stores (volume.rs:29-32), with a
// block timestamp: `block` is the offset, in blocks from the start of the next process_* call, at which the command takes
// effect — what the reference's per-block polling (processor.rs:214, volume.rs:92, sampler.rs:331) gives a host that calls
// once per block. The stream side splits the call there.
struct NodeParams;
enum CmdKind : uint32_t {
    CMD_SAMPLER = 0,   // a = SmpMsgKind, x / y / b = payload (NodeToProcessorMsg sampler.rs:21-28)
    CMD_TARGET = 1,    // a = smoothed-parameter index of the node (0: raw_gain / gain_l, 1: gain_r), f[0] = value
    CMD_COEFFS = 2,    // a = stage, f[0 .. coeff_width(kind)) = that stage's biquad or SVF coefficients (see NodeParams::coeffs)
    CMD_RS_SET = 3,    // b = resource, x = step (Q32.32), a = flags (bit0 playing, bit1 loop)
    CMD_RS_SEEK = 4,   // x = position in frames
    CMD_UPLOAD = 5     // a whole parameter array at once (set_percent_volumes, set_all_coeffs ...): a = array (0 / 1: smoothed target 0 / 1,
                       // 2: coefficient table), x = float* snapshot taken by the main thread (handed back through Channels::to_free), y = floats
};
struct Cmd { uint32_t kind, block, voice /* or FW_ALL_VOICES */, a, b, pad; uint64_t x, y; float f[6]; const NodeParams* node; };

// ---- node parameters (main-thread side; the stream side snapshots them at call start) -------
struct NodeParams {
    uint32_t kind = FW_NODE_DUMMY;
    uint32_t num_voices = 1;
    // The arrays below are the MAIN THREAD's view of the parameters: they seed the device state at activation. Once the context is
    // active every store also travels through the command ring, in program order — the stream side never reads these arrays.
    std::shared_ptr<CustomNode> custom;  // kind == FW_NODE_CUSTOM
    // volume (volume.rs:8-34)
    std::vector<float> percent, raw_gain;
    // pan
    std::vector<float> pan, gain_l, gain_r;
    // hard clip (hard_clip.rs:8-12)
    float threshold_gain = 0.0f;
    // biquad and SVF (spec ours): [voice][stage][coeff_width(kind)], a biquad stage {b0, b1, b2, a1, a2}, an SVF stage
    // {a1, a2, a3, m0, m1, m2}
    uint32_t num_stages = 0;
    std::vector<float> coeffs;
    // delay
    uint32_t delay = 0;
    // conv reverb
    uint32_t ir_len = 0, ir_channels = 0;
    std::vector<float> ir;  // [ch][len] f32 (rounded to bf16 on the device side)
    // polyphase resampler (spec ours): table [phases][taps]; the per-voice transport travels as commands
    uint32_t rs_phases = 0, rs_taps = 0; std::vector<float> rs_table;
    // sampler (sampler.rs:46-181): node-side state per voice (main thread only). `percent` / `raw_gain` above double as the
    // sampler's volume (sampler.rs:49-50). Messages travel through the context's command ring.
    bool smp_active = false;               // ActiveState is Some (sampler.rs:198-215)
    std::vector<uint8_t> smp_playing;      // SamplerNode::playing (sampler.rs:51)
    std::vector<uint16_t> smp_pending;     // messages queued per voice since the stream side last drained (ring capacity 128, sampler.rs:14)
    std::vector<uint32_t> smp_pending_epoch;  // drain epoch `smp_pending[v]` was counted in
};

// The data-plane step that runs a node (Plan::Step in runtime.cu)
enum StepKind : uint8_t { STEP_PROG, STEP_SAMPLER, STEP_TEMPORAL, STEP_REVERB, STEP_SUM, STEP_RESAMPLER, STEP_CUSTOM };

// What a node kind is, for the graph, the activation and the device lowering: one row per fw_node_kind (graph.cpp).
struct NodeKind {
    uint32_t kind; const char* name;  // name: the debug_name the graph reports
    fw_audio_node_info info;          // AudioNodeInfo (node.rs:57-79 as filled in by each basic node); out_silence_rule is unused
    uint32_t coeff_width;             // floats per stage in NodeParams::coeffs (0: no coefficient table)
    using Target = std::vector<float> NodeParams::*;
    Target target[2];                 // the target arrays of the node's smoothed parameters, in smoother order (null: none)
    StepKind step;                    // the data-plane step that runs the node (a 1-port SumNode is a copy: a PROG step)
    struct {
        bool on; ChainOpKind kind;    // the node is one chain op of this kind
        uint32_t c_in, c_out;         // the op's program widths in the generic lowering
        bool pairs;                   // the generic lowering runs the op per channel pair
        bool mask;                    // the op's body branches on the input silence mask (a stereo Volume's does not)
        bool fuses;                   // a stereo node joins fused runs of the generic lowering
    } op;
    bool per_channel_state;           // device state sized by the port count: the node is activated again when the count changes
    bool call_varying;                // kernel arguments change from call to call (cursors, positions, plugin calls): no graph replay
    bool reads_resources;             // reads the context's sample resources
};
// The row of `kind`; an unknown kind's row for an out-of-range value
const NodeKind& node_kind(uint32_t kind);
inline uint32_t coeff_width(uint32_t kind) { return node_kind(kind).coeff_width; }

// AudioNode::activate argument checks (volume.rs:63-65, sum.rs:27-29, hard_clip.rs:37-39, ours). "" => Ok.
std::string node_check_activation(const NodeParams& p, uint32_t num_inputs, uint32_t num_outputs);

struct EdgeRec { Id id; Id src, dst; uint32_t src_port = 0, dst_port = 0; };
struct NodeRec {
    Id id; uint32_t num_inputs = 0, num_outputs = 0;
    std::shared_ptr<NodeParams> params;
    bool activated = false;  // Q5: the reference never sets this to true; kept for fidelity
};

struct InAssign { uint32_t buffer; bool should_clear; uint32_t generation; Id producer; uint32_t producer_port; };
struct OutAssign { uint32_t buffer; uint32_t generation; };
struct SchedNode { Id id; std::vector<InAssign> in; std::vector<OutAssign> out; };
struct Schedule { std::vector<SchedNode> nodes; uint32_t num_buffers = 0; uint32_t max_block_frames = 0; };

struct CompileError { int code = FW_COMPILE_OK; Id node; uint32_t port = 0; std::string message; };

class Graph {
  public:
    Graph(uint32_t num_graph_inputs, uint32_t num_graph_outputs, uint32_t num_voices);

    Id graph_in() const { return gin_; }
    Id graph_out() const { return gout_; }
    Id add_node(uint32_t n_in, uint32_t n_out, std::shared_ptr<NodeParams> p);
    bool remove_node(Id id, std::vector<Id>* removed_edges);
    bool set_num_inputs(Id id, uint32_t n, std::vector<Id>* removed_edges);
    bool set_num_outputs(Id id, uint32_t n, std::vector<Id>* removed_edges);
    int connect(Id src, uint32_t sp, Id dst, uint32_t dp, bool check_cycles, Id* out_edge);
    bool disconnect(Id src, uint32_t sp, Id dst, uint32_t dp);
    bool disconnect_edge(Id edge);
    const EdgeRec* edge(Id e) const { return edges_.find(e); }
    NodeRec* node(Id n) { return nodes_.find(n); }
    uint32_t num_nodes() const { return nodes_.size(); }
    uint32_t num_edges() const { return edges_.size(); }
    template <class F> void each_node(F&& f) { nodes_.each(f); }
    template <class F> void each_edge(F&& f) { edges_.each(f); }
    bool cycle_detected();
    void reset();
    bool needs_compile() const { return dirty_; }
    void mark_dirty() { dirty_ = true; }
    void clear_dirty() { dirty_ = false; }

    // compiler.rs:139-152: topological order + buffer assignment
    CompileError compile_schedule(uint32_t max_block_frames, Schedule* out);

    // bookkeeping used by the context (graph.rs:119-121)
    std::vector<Id> nodes_to_activate, nodes_removed_since_compile;

  private:
    bool topo_order(std::vector<Id>* order);  // false => cycle
    void drop_edges_into(Id node, uint32_t port, std::vector<Id>* removed);
    void drop_edges_from(Id node, uint32_t port, std::vector<Id>* removed);
    static uint64_t port_key(Id n, uint32_t port) { return ((uint64_t)n.slot << 40) ^ ((uint64_t)n.gen << 8) ^ port; }
    struct EdgeKey { uint64_t a, b; bool operator==(const EdgeKey& o) const { return a == o.a && b == o.b; } };
    struct EdgeKeyHash { size_t operator()(const EdgeKey& k) const { return std::hash<uint64_t>()(k.a * 0x9E3779B97F4A7C15ull ^ k.b); } };
    static EdgeKey edge_key(Id s, uint32_t sp, Id d, uint32_t dp) { return EdgeKey{s.pack() ^ ((uint64_t)sp << 56), d.pack() ^ ((uint64_t)dp << 56)}; }

    SlotTable<NodeRec> nodes_;
    SlotTable<EdgeRec> edges_;
    std::unordered_set<uint64_t> connected_inputs_;        // (dst node, dst port)
    std::unordered_map<EdgeKey, Id, EdgeKeyHash> by_ends_; // existing edges
    Id gin_, gout_;
    bool dirty_ = true;
    uint32_t num_voices_;
};

// ---- isomorphic-voice detection (SURVEY §8 f2; voices.cpp) --------------------------------------------------------------------
// The reference runs ONE graph; a mixer of V identical voices is V copies of a sub-graph feeding a tree of SumNodes in front of
// graph_out. This recognises that shape in a flat graph, so that it can be run as `num_voices = V` instances of one voice graph with
// a master bus — bit-identical, because the bus IS that tree (DESIGN.md "Batching extension"): level l adds neighbours (2i, 2i+1)
// with a 2-port SumNode (2C inputs -> C outputs, sum.rs:69-81), an unpaired last element goes through a 1-port SumNode
// (C -> C, the copy path sum.rs:58-65).
struct VoiceDetection {
    uint32_t num_voices = 0, voice_inputs = 0, voice_outputs = 0;
    std::vector<std::vector<Id>> nodes;      // [template node, canonical order][voice]
    struct Src { int node = -1; uint32_t port = 0; };  // node >= 0: template node; -1: unconnected; -2: graph_in, port = channel of the voice
    std::vector<std::vector<Src>> inputs;    // [template node][input port]
    std::vector<Src> outputs;                // [voice output channel]: what feeds the bus
    std::vector<Id> tree;                    // the SumNodes of the bus tree (they disappear into master_bus = 1)
};
// The deepest reading of the SumNode tree in front of graph_out whose leaves are disjoint isomorphic voices wins; a graph that is
// simply one voice answers true with num_voices == 1 (then *why says why a deeper reading was rejected, if there was a tree).
// false + *why: not even that (e.g. side branches that never reach graph_out).
bool detect_voices(Graph& g, VoiceDetection* out, std::string* why);

}  // namespace fw
