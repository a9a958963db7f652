// graph.cpp — see graph.hpp. Behaviour follows firewheel-graph's graph.rs / compiler.rs
// (file:line cited per function); the data structures are this project's own.
#include "graph.hpp"

#include <algorithm>

namespace fw {

// One row per fw_node_kind in kind order, then the row of an unknown kind. info: {min in, max in, min out, max out, updates}; op: {on,
// kind, c_in, c_out, pairs, mask, fuses}, {} when the node is not a chain op; chan, vary, res: per_channel_state, call_varying, reads_resources.
static constexpr NodeKind kNodeKinds[] = {
    //kind                   name              info               coeffs targets                                     step            op                                        chan   vary   res
    {FW_NODE_DUMMY,          "dummy",          {0, 64, 0, 64, 0}, 0,     {},                                         STEP_PROG,      {},                                       false, false, false},  // dummy.rs:8-18
    {FW_NODE_VOLUME,         "volume",         {1, 64, 1, 64, 0}, 0,     {&NodeParams::raw_gain},                    STEP_PROG,      {true, OP_GAIN, 2, 2, true, true, true},  false, false, false},  // volume.rs:43-54
    {FW_NODE_SUM,            "sum",            {1, 64, 1, 64, 0}, 0,     {},                                         STEP_SUM,       {},                                       false, false, false},  // sum.rs:7
    {FW_NODE_MONO_TO_STEREO, "mono_to_stereo", {1, 1, 2, 2, 0},   0,     {},                                         STEP_PROG,      {true, OP_M2S, 1, 2, false, true, false}, false, false, false},  // mono_to_stereo.rs:7-18
    {FW_NODE_STEREO_TO_MONO, "stereo_to_mono", {2, 2, 1, 1, 0},   0,     {},                                         STEP_PROG,      {true, OP_S2M, 2, 1, false, true, false}, false, false, false},  // stereo_to_mono.rs:7-18
    {FW_NODE_HARD_CLIP,      "hard_clip",      {1, 64, 1, 64, 0}, 0,     {},                                         STEP_PROG,      {true, OP_CLIP, 2, 2, true, true, false}, false, false, false},  // hard_clip.rs:17
    {FW_NODE_PAN,            "pan",            {2, 2, 2, 2, 0},   0,     {&NodeParams::gain_l, &NodeParams::gain_r}, STEP_PROG,      {true, OP_PAN, 2, 2, false, false, true}, false, false, false},
    {FW_NODE_BIQUAD,         "biquad",         {1, 64, 1, 64, 0}, 5,     {},                                         STEP_TEMPORAL,  {},                                       true,  false, false},
    {FW_NODE_DELAY,          "delay",          {1, 64, 1, 64, 0}, 0,     {},                                         STEP_TEMPORAL,  {},                                       true,  true,  false},
    {FW_NODE_CONV_REVERB,    "conv_reverb",    {1, 64, 1, 64, 0}, 0,     {},                                         STEP_REVERB,    {},                                       true,  true,  false},
    {FW_NODE_SAMPLER,        "beep_test",      {0, 0, 1, 64, 1},  0,     {&NodeParams::raw_gain},                    STEP_SAMPLER,   {},                                       false, false, true},   // Q8: sampler.rs:186 really says that; sampler.rs:189-196
    {FW_NODE_SVF,            "svf",            {1, 64, 1, 64, 0}, 6,     {},                                         STEP_TEMPORAL,  {},                                       true,  false, false},
    {FW_NODE_RESAMPLER,      "resampler",      {0, 0, 1, 64, 0},  0,     {},                                         STEP_RESAMPLER, {},                                       false, true,  true},
    {FW_NODE_CUSTOM,         "custom",         {1, 64, 1, 64, 0}, 0,     {},                                         STEP_CUSTOM,    {},                                       false, true,  false},  // the context reports the plugin's own name and info
    {FW_NODE_CUSTOM + 1,     "unknown",        {1, 64, 1, 64, 0}, 0,     {},                                         STEP_PROG,      {},                                       false, false, false},
};
constexpr bool rows_in_kind_order() { for (uint32_t k = 0; k < sizeof(kNodeKinds) / sizeof(kNodeKinds[0]); ++k) if (kNodeKinds[k].kind != k) return false; return true; }
static_assert(sizeof(kNodeKinds) / sizeof(kNodeKinds[0]) == FW_NODE_CUSTOM + 2 && rows_in_kind_order(), "one row per fw_node_kind, then the unknown row");

const NodeKind& node_kind(uint32_t kind) { return kNodeKinds[kind <= FW_NODE_CUSTOM ? kind : FW_NODE_CUSTOM + 1]; }

std::string node_check_activation(const NodeParams& p, uint32_t ni, uint32_t no) {
    auto got = [&] { return "Got num_inputs: " + std::to_string(ni) + ", num_outputs: " + std::to_string(no); };
    switch (p.kind) {
        case FW_NODE_VOLUME:  // volume.rs:63-65
            if (ni != no) return "The number of inputs on a VolumeNode node must equal the number of outputs. " + got();
            break;
        case FW_NODE_SUM:  // sum.rs:27-29
            if (no == 0 || ni % no != 0) return "The number of inputs on a SumNode must be a multiple of the number of outputs. " + got();
            break;
        case FW_NODE_HARD_CLIP:  // hard_clip.rs:37-39
            if (ni != no) return "The number of inputs on a HardClip node must equal the number of outputs. " + got();
            break;
        case FW_NODE_PAN:
            if (ni != 2 || no != 2) return "A PanNode must have 2 inputs and 2 outputs. " + got();
            break;
        case FW_NODE_BIQUAD:
            if (ni != no) return "The number of inputs on a BiquadNode must equal the number of outputs. " + got();
            break;
        case FW_NODE_DELAY:
            if (ni != no) return "The number of inputs on a DelayNode must equal the number of outputs. " + got();
            break;
        case FW_NODE_SVF:
            if (ni != no) return "The number of inputs on an SvfNode must equal the number of outputs. " + got();
            break;
        case FW_NODE_RESAMPLER:
            if (no == 0 || p.rs_phases == 0 || p.rs_phases > 1024 || (p.rs_phases & (p.rs_phases - 1)) || p.rs_taps < 2 || p.rs_taps > 64 || (p.rs_taps & 1))
                return "A ResamplerNode needs >= 1 output, a power-of-two phase count <= 1024 and an even tap count <= 64.";
            break;
        case FW_NODE_CONV_REVERB:
            if (ni != no || p.ir_len == 0 || p.ir_channels == 0)
                return "A ConvReverbNode needs num_inputs == num_outputs and a non-empty IR. " + got();
            break;
        default: break;
    }
    return "";
}

Graph::Graph(uint32_t n_gin, uint32_t n_gout, uint32_t num_voices) : num_voices_(num_voices) {
    // graph.rs:125-168: graph_in = Dummy(0 -> n), graph_out = Dummy(n -> 0); both queued for activation
    auto mk = [&](uint32_t ni, uint32_t no) {
        auto p = std::make_shared<NodeParams>();
        p->kind = FW_NODE_DUMMY; p->num_voices = num_voices;
        NodeRec r; r.num_inputs = ni; r.num_outputs = no; r.params = p;
        Id id = nodes_.insert(std::move(r));
        nodes_.find(id)->id = id;
        return id;
    };
    gin_ = mk(0, n_gin);
    gout_ = mk(n_gout, 0);
    nodes_to_activate = {gin_, gout_};
}

Id Graph::add_node(uint32_t ni, uint32_t no, std::shared_ptr<NodeParams> p) {  // graph.rs:201-231
    NodeRec r; r.num_inputs = ni; r.num_outputs = no; r.params = std::move(p);
    Id id = nodes_.insert(std::move(r));
    nodes_.find(id)->id = id;
    nodes_to_activate.push_back(id);
    dirty_ = true;
    return id;
}

void Graph::drop_edges_into(Id node, uint32_t port, std::vector<Id>* removed) {  // graph.rs:531-550
    std::vector<Id> hit;
    edges_.each([&](Id eid, EdgeRec& e) { if (e.dst == node && e.dst_port == port) hit.push_back(eid); });
    for (Id e : hit) disconnect_edge(e);
    if (removed) removed->insert(removed->end(), hit.begin(), hit.end());
}
void Graph::drop_edges_from(Id node, uint32_t port, std::vector<Id>* removed) {  // graph.rs:552-571
    std::vector<Id> hit;
    edges_.each([&](Id eid, EdgeRec& e) { if (e.src == node && e.src_port == port) hit.push_back(eid); });
    for (Id e : hit) disconnect_edge(e);
    if (removed) removed->insert(removed->end(), hit.begin(), hit.end());
}

bool Graph::remove_node(Id id, std::vector<Id>* removed) {  // graph.rs:268-299
    if (id == gin_ || id == gout_) return false;
    NodeRec rec;
    if (!nodes_.erase(id, &rec)) return false;
    for (uint32_t p = 0; p < rec.num_inputs; ++p) drop_edges_into(id, p, removed);
    for (uint32_t p = 0; p < rec.num_outputs; ++p) drop_edges_from(id, p, removed);
    for (uint32_t p = 0; p < rec.num_inputs; ++p) connected_inputs_.erase(port_key(id, p));
    nodes_removed_since_compile.push_back(id);
    dirty_ = true;
    return true;
}

bool Graph::set_num_inputs(Id id, uint32_t n, std::vector<Id>* removed) {  // graph.rs:315-343
    if (id == gin_) return false;
    NodeRec* r = nodes_.find(id);
    if (!r) return false;
    uint32_t old = r->num_inputs;
    for (uint32_t p = n; p < old; ++p) { drop_edges_into(id, p, removed); connected_inputs_.erase(port_key(id, p)); }
    nodes_.find(id)->num_inputs = n;
    dirty_ = true;
    return true;
}
bool Graph::set_num_outputs(Id id, uint32_t n, std::vector<Id>* removed) {  // graph.rs:349-375
    if (id == gout_) return false;
    NodeRec* r = nodes_.find(id);
    if (!r) return false;
    uint32_t old = r->num_outputs;
    for (uint32_t p = n; p < old; ++p) drop_edges_from(id, p, removed);
    nodes_.find(id)->num_outputs = n;
    dirty_ = true;
    return true;
}

int Graph::connect(Id src, uint32_t sp, Id dst, uint32_t dp, bool check_cycles, Id* out_edge) {  // graph.rs:396-477
    const NodeRec* s = nodes_.find(src);
    if (!s) return FW_EDGE_SRC_NODE_NOT_FOUND;
    const NodeRec* d = nodes_.find(dst);
    if (!d) return FW_EDGE_DST_NODE_NOT_FOUND;
    if (sp >= s->num_outputs) return FW_EDGE_OUT_PORT_OUT_OF_RANGE;
    if (dp >= d->num_inputs) return FW_EDGE_IN_PORT_OUT_OF_RANGE;
    if (src == dst) return FW_EDGE_CYCLE_DETECTED;
    EdgeKey k = edge_key(src, sp, dst, dp);
    if (by_ends_.count(k)) return FW_EDGE_ALREADY_EXISTS;
    if (!connected_inputs_.insert(port_key(dst, dp)).second) return FW_EDGE_INPUT_PORT_ALREADY_CONNECTED;
    EdgeRec e; e.src = src; e.dst = dst; e.src_port = sp; e.dst_port = dp;
    Id eid = edges_.insert(e);
    edges_.find(eid)->id = eid;
    by_ends_[k] = eid;
    if (check_cycles && cycle_detected()) {
        // Faithful to graph.rs:466-472 (SURVEY Q9): only the edge record is rolled back; the
        // by-ends map and the connected-port set keep their entries.
        edges_.erase(eid);
        return FW_EDGE_CYCLE_DETECTED;
    }
    dirty_ = true;
    if (out_edge) *out_edge = eid;
    return FW_EDGE_OK;
}

bool Graph::disconnect(Id src, uint32_t sp, Id dst, uint32_t dp) {  // graph.rs:483-501
    auto it = by_ends_.find(edge_key(src, sp, dst, dp));
    if (it == by_ends_.end()) return false;
    Id eid = it->second;
    by_ends_.erase(it);
    disconnect_edge(eid);
    return true;
}
bool Graph::disconnect_edge(Id eid) {  // graph.rs:507-524
    EdgeRec e;
    if (!edges_.erase(eid, &e)) return false;
    by_ends_.erase(edge_key(e.src, e.src_port, e.dst, e.dst_port));
    connected_inputs_.erase(port_key(e.dst, e.dst_port));
    dirty_ = true;
    return true;
}

void Graph::reset() {  // graph.rs:171-182
    std::vector<Id> ids;
    nodes_.each([&](Id id, NodeRec&) { if (id != gin_ && id != gout_) ids.push_back(id); });
    for (Id id : ids) remove_node(id, nullptr);
}

// Kahn's algorithm over slots (compiler.rs:232-300): graph_in seeds the queue, then every
// other source node in ascending slot order; graph_out is withheld and appended last.
bool Graph::topo_order(std::vector<Id>* order) {
    uint32_t nslots = nodes_.slot_count();
    std::vector<int32_t> indeg(nslots, 0);
    std::vector<std::vector<uint32_t>> succ(nslots);  // successor slots in edge-slot order, one entry per edge
    std::vector<uint8_t> has_in(nslots, 0);
    edges_.each([&](Id, EdgeRec& e) {
        indeg[e.dst.slot] += 1; has_in[e.dst.slot] = 1;
        succ[e.src.slot].push_back(e.dst.slot);
    });
    std::deque<uint32_t> q;
    q.push_back(gin_.slot);
    nodes_.each([&](Id id, NodeRec&) { if (!has_in[id.slot] && id.slot != gin_.slot) q.push_back(id.slot); });
    uint32_t visited = 0;
    while (!q.empty()) {
        uint32_t s = q.front(); q.pop_front();
        ++visited;
        for (uint32_t d : succ[s]) if (--indeg[d] == 0) q.push_back(d);
        if (order && s != gout_.slot) { Id id; nodes_.by_slot(s, &id); order->push_back(id); }
    }
    if (order) order->push_back(gout_);
    return visited == nodes_.size();
}

bool Graph::cycle_detected() { return !topo_order(nullptr); }  // compiler.rs:154-168

CompileError Graph::compile_schedule(uint32_t max_block_frames, Schedule* out) {
    CompileError err;
    std::vector<Id> order;
    if (!topo_order(&order)) { err.code = FW_COMPILE_CYCLE_DETECTED; return err; }  // compiler.rs:295-297

    // Per-node port tables in edge-slot order.
    uint32_t nslots = nodes_.slot_count();
    struct PortEdge { Id edge; uint32_t port; Id other; uint32_t other_port; };
    std::vector<std::vector<PortEdge>> incoming(nslots), outgoing(nslots);
    edges_.each([&](Id eid, EdgeRec& e) {
        incoming[e.dst.slot].push_back(PortEdge{eid, e.dst_port, e.src, e.src_port});
        outgoing[e.src.slot].push_back(PortEdge{eid, e.src_port, e.dst, e.dst_port});
    });

    // Buffer assignment (compiler.rs:302-412). A buffer returns to the LIFO free stack when the
    // last edge holding it has been consumed; it is only recycled after the consuming node's own
    // ports have all been assigned, so a node never sees aliased buffers.
    struct Buf { uint32_t idx, generation, holders; };
    std::vector<Buf> live;                       // indexed by handle
    std::vector<std::pair<uint32_t, uint32_t>> free_stack;  // (idx, generation)
    uint32_t count = 0;
    auto acquire = [&]() -> uint32_t {
        Buf b{0, 0, 0};
        if (!free_stack.empty()) { b.idx = free_stack.back().first; b.generation = free_stack.back().second; free_stack.pop_back(); }
        else { b.idx = count++; b.generation = 0; }
        live.push_back(b);
        return (uint32_t)live.size() - 1;
    };
    std::unordered_map<uint64_t, uint32_t> edge_buf;  // edge id -> handle

    out->nodes.clear();
    out->max_block_frames = max_block_frames;
    for (Id nid : order) {
        NodeRec& nr = *nodes_.find(nid);
        SchedNode sn; sn.id = nid;
        std::vector<uint32_t> release;  // handles, in port order; each entry drops one holder
        for (uint32_t port = 0; port < nr.num_inputs; ++port) {
            const PortEdge* hit = nullptr; uint32_t n_hit = 0;
            for (const PortEdge& pe : incoming[nid.slot]) if (pe.port == port) { if (!hit) hit = &pe; ++n_hit; }
            if (n_hit == 0) {
                uint32_t h = acquire(); live[h].holders = 1;
                sn.in.push_back(InAssign{live[h].idx, true, live[h].generation, Id{}, 0});
                release.push_back(h);
            } else if (n_hit == 1) {
                uint32_t h = edge_buf.at(hit->edge.pack());
                edge_buf.erase(hit->edge.pack());
                sn.in.push_back(InAssign{live[h].idx, false, live[h].generation, hit->other, hit->other_port});
                release.push_back(h);
            } else {
                err.code = FW_COMPILE_MANY_TO_ONE; err.node = nid; err.port = port;  // compiler.rs:363-365
                return err;
            }
        }
        for (uint32_t port = 0; port < nr.num_outputs; ++port) {
            uint32_t h = acquire(), n_out_edges = 0;
            for (const PortEdge& pe : outgoing[nid.slot]) if (pe.port == port) { edge_buf[pe.edge.pack()] = h; ++n_out_edges; }
            sn.out.push_back(OutAssign{live[h].idx, live[h].generation});
            if (n_out_edges == 0) { live[h].holders = 1; release.push_back(h); }
            else live[h].holders = n_out_edges;
        }
        for (uint32_t h : release)
            if (--live[h].holders == 0) free_stack.emplace_back(live[h].idx, live[h].generation + 1);
        out->nodes.push_back(std::move(sn));
    }
    out->num_buffers = count;
    return err;
}

}  // namespace fw
