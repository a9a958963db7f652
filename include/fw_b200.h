/* fw_b200.h — C ABI of firewheel-b200: the drop-in boundary for the per-block
 * audio-graph DSP path of BillyDM/firewheel @ 2dfa7ea.
 *
 * Every entry point names the reference interface it replaces (file:line relative
 * to the reference tree). A Rust `-sys` crate binds these 1:1 (INTEGRATION.md).
 * Plain pointers and sizes only; no exceptions or panics cross this boundary.
 *
 * The SAME declarations are exported twice:
 *   libfirewheel_b200.so   prefix fw_   — the product: CUDA sm_90a, no CPU fallback
 *   oracle/_build/libfw_oracle.so  prefix fwo_  — CPU oracle (test infrastructure only)
 * so parity tests drive both through identical code (FW_API_PREFIX selects).
 *
 * Batching extension over the reference: a context holds `num_voices` instances
 * of one voice graph (same topology, per-voice parameters and state). With
 * `master_bus = 1` the graph_out channels of all voices are mixed by a balanced
 * binary tree of 2-port SumNodes (sum.rs:69-81) — level l adds neighbours
 * (2i, 2i+1); an unpaired last element is carried up unchanged (the 1-port
 * SumNode copy path, sum.rs:58-65). Each graph_out channel has its own tree, so
 * the bus takes 1 to FW_MAX_BUS_CHANNELS graph_out channels (mono through 7.1);
 * the device refuses a wider bus at compile time (FW_COMPILE_UNSUPPORTED_ON_DEVICE).
 * num_voices = 1, master_bus = 0 is exactly the reference.
 *
 * Buffer layouts (f32):
 *   interleaved in : [voice][frames][n_in]      out: [voice][frames][n_out]  (master bus: [frames][n_out])
 *   planar      in : [voice][n_in][frames]      out: [voice][n_out][frames]  (master bus: [n_out][frames])
 */
#ifndef FW_B200_H
#define FW_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#ifndef FW_API_PREFIX
#define FW_API_PREFIX fw_
#endif
#define FW_CAT2(a, b) a##b
#define FW_CAT(a, b) FW_CAT2(a, b)
#define FW_FN(name) FW_CAT(FW_API_PREFIX, name)
#define FW_EXPORT __attribute__((visibility("default")))

/* NodeID / EdgeID: thunderdome generational index (graph.rs:20-23, compiler.rs:63)
 * packed as slot | generation << 32. */
typedef uint64_t fw_node_id;
typedef uint64_t fw_edge_id;
#define FW_ID_DANGLING UINT64_MAX
#define FW_ALL_VOICES UINT32_MAX
#define FW_MAX_PORTS 64u /* node.rs:62,70; compiler.rs:202-203 */
#define FW_MAX_BUS_CHANNELS 8u /* graph_out channels of a master bus on the device (7.1, the most HDMI LPCM carries) */

typedef struct fw_ctx fw_ctx;             /* FirewheelGraphCtx   context.rs:29 */
typedef struct fw_processor fw_processor; /* FirewheelProcessor  processor.rs:18 */

/* AudioGraphConfig (graph.rs:91-107) + batching fields */
typedef struct fw_graph_config {
    uint32_t num_graph_inputs;      /* default 0 */
    uint32_t num_graph_outputs;     /* default 2 */
    uint32_t initial_node_capacity; /* default 64 */
    uint32_t initial_edge_capacity; /* default 256 */
    uint32_t num_voices;            /* >= 1 */
    uint32_t master_bus;            /* 0 | 1 */
    int32_t device;                 /* CUDA ordinal (ignored by the oracle) */
    uint32_t max_call_frames;       /* product: all per-call device memory is reserved at activate / update for stretches of this many
                                       frames (0 = 64 blocks of max_block_frames); a longer process_* call is processed as consecutive
                                       chunks — same samples, more launches. The stream side never allocates. */
} fw_graph_config;

/* Built-in node kinds. The Rust side constructs `impl Into<Box<dyn AudioNode>>`
 * values (graph.rs:201-206); over the C ABI a node is described by value. */
enum fw_node_kind {
    FW_NODE_DUMMY = 0,          /* basic_nodes/dummy.rs */
    FW_NODE_VOLUME = 1,         /* basic_nodes/volume.rs  f0 = percent_volume */
    FW_NODE_SUM = 2,            /* basic_nodes/sum.rs */
    FW_NODE_MONO_TO_STEREO = 3, /* basic_nodes/mono_to_stereo.rs */
    FW_NODE_STEREO_TO_MONO = 4, /* basic_nodes/stereo_to_mono.rs */
    FW_NODE_HARD_CLIP = 5,      /* basic_nodes/hard_clip.rs  f0 = threshold_db */
    FW_NODE_PAN = 6,            /* spec ours (SURVEY §8 a10)  f0 = pan in [-1,1] */
    FW_NODE_BIQUAD = 7,         /* spec ours (a11)  u0 = num_stages (<= 8) */
    FW_NODE_DELAY = 8,          /* spec ours (a12)  u0 = delay in frames */
    FW_NODE_CONV_REVERB = 9,    /* spec ours (a14)  u0 = ir_len, u1 = ir_channels, data = IR [ch][len] */
    FW_NODE_SAMPLER = 10,       /* basic_nodes/sampler.rs  f0 = percent_volume; 0 inputs, 1..64 outputs */
    FW_NODE_SVF = 11,           /* spec ours (a11)  u0 = num_stages (<= 8): trapezoidal state-variable filter cascade */
    FW_NODE_RESAMPLER = 12,     /* spec ours (a13)  polyphase-resampling sample player: u0 = phases P (power of two, <= 1024),
                                   u1 = taps T (even, <= 64), data = Kaiser-windowed-sinc table [P][T]; 0 inputs, 1..64 outputs */
    FW_NODE_CUSTOM = 13         /* a user node behind fw_node_vtable (graph_add_custom_node); never passed in a fw_node_desc */
};
/* SampleResource implementations (firewheel-core/src/sample_resource.rs:28-335). Interleaved data is [frame][ch],
 * planar ("Vec<Vec<T>>") is [ch][frame]. */
enum fw_sample_format {
    FW_SAMPLE_F32_PLANAR = 0,       /* Vec<Vec<f32>>            :249-266 */
    FW_SAMPLE_F32_INTERLEAVED = 1,  /* InterleavedResourceF32   :142-197 */
    FW_SAMPLE_I16_INTERLEAVED = 2,  /* InterleavedResourceI16   :28-83,  pcm_i16_to_f32 :337 */
    FW_SAMPLE_U16_INTERLEAVED = 3,  /* InterleavedResourceU16   :85-140, pcm_u16_to_f32 :342 */
    FW_SAMPLE_I16_PLANAR = 4,       /* Vec<Vec<i16>>            :199-222 */
    FW_SAMPLE_U16_PLANAR = 5        /* Vec<Vec<u16>>            :224-247 */
};
/* LoopRange (sampler.rs:16-19) as passed to sampler_set_loop_range */
enum fw_loop_mode { FW_LOOP_NONE = 0, FW_LOOP_FULL = 1, FW_LOOP_RANGE_SECS = 2 };
/* sampler_* return codes: Ok(()) => 0; Err(()) from a full message ring (capacity 128, sampler.rs:14) => -2 */
enum fw_sampler_status { FW_SAMPLER_OK = 0, FW_SAMPLER_NOT_A_SAMPLER = -1, FW_SAMPLER_RING_FULL = -2,
                         FW_SAMPLER_NOT_ACTIVATED = -3 /* the reference hits todo!() */, FW_SAMPLER_BAD_ARGS = -4 };
typedef struct fw_node_desc {
    uint32_t kind;
    uint32_t u0, u1, u2;
    float f0, f1, f2, f3;
    const float* data;
    uint64_t data_len; /* floats */
} fw_node_desc;

/* ---- the plugin boundary: trait AudioNode / trait AudioNodeProcessor (firewheel-core/src/node.rs:6-53) as a C vtable ----------
 * A Rust `Box<dyn AudioNode>` crosses the boundary as (vtable, node). The graph owns the node: `drop_node` runs when it is
 * removed or the context is freed (Box drop). Differences forced by batching, all stated here:
 *   * one node object serves all `num_voices` voices: `activate` is called ONCE per activation and returns ONE processor for
 *     all voices (the reference: one processor per node, graph.rs:596-602);
 *   * the processor has two forms of `process`. `process` is the reference's signature plus the voice index — the CPU oracle
 *     calls it per voice and per block. `process_device` is what the product calls: all voices and all blocks of a call at
 *     once, device pointers, on the processor's CUDA stream; the plugin enqueues its own kernels there and returns. A node
 *     without `process_device` cannot run on the product: the graph then fails to compile with FW_COMPILE_UNSUPPORTED_ON_DEVICE
 *     (there is no CPU fallback);
 *   * ProcInfo::out_silence_mask is "an optional optimization hint" (node.rs:100-106). On the device the control plane runs ahead
 *     of the samples, so a custom node DECLARES its hint as a rule in `info` instead of computing it from data; the oracle
 *     checks that what `process` writes equals the declared rule. FW_OUT_SILENCE_NONE (the ProcInfo default) is always valid.
 * Calls: debug_name / info / activate / deactivate / update / drop_* on the main thread (AudioNode is not Send); process* on the
 * stream thread (AudioNodeProcessor: Send). `deactivate(node, processor)` is called where the reference calls
 * `deactivate(Some(processor))`: activation roll-back (graph.rs:603-609) and a node removed while active (graph.rs:644-648);
 * otherwise a processor is dropped with `drop_processor` (the reference never sets `activated`, SURVEY Q5). */
typedef struct fw_audio_node_info { /* AudioNodeInfo node.rs:57-79 */
    uint32_t num_min_supported_inputs, num_max_supported_inputs;
    uint32_t num_min_supported_outputs, num_max_supported_outputs;
    uint32_t updates;            /* call `update` from ctx_update (graph.rs:691-697) */
    uint32_t out_silence_rule;   /* fw_out_silence_rule */
} fw_audio_node_info;
enum fw_out_silence_rule {
    FW_OUT_SILENCE_NONE = 0,               /* no output is ever flagged (ProcInfo default, node.rs:104-106) */
    FW_OUT_SILENCE_PASSTHROUGH = 1,        /* output i flagged iff input i flagged (num_inputs == num_outputs; VolumeNode's rule, volume.rs:110) */
    FW_OUT_SILENCE_ALL_IF_ALL_INPUTS = 2   /* every output flagged iff every input is flagged (SumNode's rule, sum.rs:52-56) */
};
typedef struct fw_proc_info { /* ProcInfo node.rs:94-118 */
    uint64_t in_silence_mask;
    uint64_t* out_silence_mask;  /* starts as 0 = NONE_SILENT (processor.rs:233) */
    double stream_time_secs;
    uint32_t stream_status;      /* fw_stream_status bits */
    uint32_t reserved;
    void* user_cx;               /* cx: &mut Box<dyn Any + Send> */
} fw_proc_info;
/* One process_device call = every voice and every block of one process_* call (frames = num_blocks blocks of block_frames,
 * the last one possibly shorter). Channel i of voice v is the `frames` floats at inputs[i] + v * in_voice_stride; inputs and
 * outputs never alias (schedule.rs:365-369). in_silence_masks[k * num_voices + v] is ProcInfo::in_silence_mask of voice v in
 * block k. Everything the plugin launches must go to `cuda_stream`. */
typedef struct fw_device_block {
    uint32_t num_voices, num_inputs, num_outputs, block_frames, num_blocks, stream_status;
    uint64_t frames, in_voice_stride, out_voice_stride;
    const float* const* inputs;  /* host array of num_inputs device pointers */
    float* const* outputs;       /* host array of num_outputs device pointers */
    const uint64_t* in_silence_masks; /* device */
    double stream_time_secs;
    void* cuda_stream;           /* cudaStream_t */
    void* user_cx;
} fw_device_block;
typedef struct fw_node_vtable {
    const char* (*debug_name)(void* node);                                               /* node.rs:7 (static lifetime) */
    void (*info)(void* node, fw_audio_node_info* out);                                   /* node.rs:9 */
    /* node.rs:12-18. 0 => *out_processor set; nonzero => error text in err (Box<dyn Error>). `device` is the CUDA ordinal on the
     * product and -1 on the oracle. */
    int (*activate)(void* node, uint32_t sample_rate, uint32_t max_block_frames, uint32_t num_inputs, uint32_t num_outputs,
                    uint32_t num_voices, int32_t device, void** out_processor, char* err, uint32_t err_cap);
    void (*deactivate)(void* node, void* processor_or_null);                             /* node.rs:26; takes the processor over */
    void (*update)(void* node);                                                          /* node.rs:32 */
    void (*drop_node)(void* node);                                                       /* Box<dyn AudioNode> drop */
    void (*process)(void* processor, uint32_t voice, uint64_t frames, const float* const* inputs, uint32_t num_inputs,
                    float* const* outputs, uint32_t num_outputs, fw_proc_info* info);    /* node.rs:46-52, host slices */
    int (*process_device)(void* processor, const fw_device_block* blk);                  /* 0 on success */
    void (*drop_processor)(void* processor);                                             /* Box<dyn AudioNodeProcessor> drop */
} fw_node_vtable;

/* AddEdgeError (graph/error.rs:14-37) */
enum fw_add_edge_error {
    FW_EDGE_OK = 0,
    FW_EDGE_SRC_NODE_NOT_FOUND = 1,
    FW_EDGE_DST_NODE_NOT_FOUND = 2,
    FW_EDGE_IN_PORT_OUT_OF_RANGE = 3,
    FW_EDGE_OUT_PORT_OUT_OF_RANGE = 4,
    FW_EDGE_ALREADY_EXISTS = 5,
    FW_EDGE_INPUT_PORT_ALREADY_CONNECTED = 6,
    FW_EDGE_CYCLE_DETECTED = 7
};
/* CompileGraphError (graph/error.rs:101-116) */
enum fw_compile_error {
    FW_COMPILE_OK = 0,
    FW_COMPILE_CYCLE_DETECTED = 1,
    FW_COMPILE_NODE_ON_EDGE_NOT_FOUND = 2,
    FW_COMPILE_NODE_ID_NOT_UNIQUE = 3,
    FW_COMPILE_EDGE_ID_NOT_UNIQUE = 4,
    FW_COMPILE_MANY_TO_ONE = 5,
    FW_COMPILE_NODE_ACTIVATION_FAILED = 6,
    FW_COMPILE_MESSAGE_CHANNEL_FULL = 7,
    /* product only: the graph is valid for the reference but has no device lowering yet. The refusals: a user node without
     * process_device; a DummyAudioNode with outputs inside the graph; a MonoToStereoNode that is not 1 -> 2 or a StereoToMonoNode that
     * is not 2 -> 1; a master bus over more than FW_MAX_BUS_CHANNELS live channels (graph_out ports that are also stream channels);
     * silence flags of one voice that do not fit in one SM's shared memory (about 930 000 pool buffers on an H100). The number of nodes, buffers, ports, smoothed parameters, samplers and resamplers is not limited otherwise. */
    FW_COMPILE_UNSUPPORTED_ON_DEVICE = 100
};
/* FirewheelProcessorStatus (processor.rs:12-16) + device-error code */
enum fw_processor_status { FW_PROC_OK = 0, FW_PROC_DROP_PROCESSOR = 1, FW_PROC_DEVICE_ERROR = -1, FW_PROC_BAD_ARGS = -2 };
/* StreamStatus bitflags (node.rs:120-132) */
enum fw_stream_status { FW_STREAM_INPUT_OVERFLOW = 1, FW_STREAM_OUTPUT_UNDERFLOW = 2 };
/* UpdateStatus (context.rs:245-254) */
enum fw_update_kind { FW_UPDATE_INACTIVE = 0, FW_UPDATE_ACTIVE = 1, FW_UPDATE_DEACTIVATED = 2 };
typedef struct fw_update_status {
    int32_t kind;           /* fw_update_kind */
    int32_t graph_error;    /* fw_compile_error; FW_COMPILE_OK if none */
    fw_node_id error_node;  /* ManyToOne / NodeActivationFailed */
    uint32_t error_port;
    uint32_t reserved;
    void* returned_user_cx; /* Deactivated { returned_user_cx } */
} fw_update_status;

typedef struct fw_node_info { /* NodeEntry (compiler.rs:12-23) + AudioNodeInfo (node.rs:57-79) */
    uint32_t num_inputs, num_outputs;
    uint32_t kind;
    uint32_t num_min_supported_inputs, num_max_supported_inputs;
    uint32_t num_min_supported_outputs, num_max_supported_outputs;
    uint32_t updates;
    char debug_name[32];
} fw_node_info;
typedef struct fw_edge_info { /* Edge (compiler.rs:68-78) */
    fw_edge_id id;
    fw_node_id src_node, dst_node;
    uint32_t src_port, dst_port;
} fw_edge_info;
/* ScheduledNode (schedule.rs:13-30): debugging / visualisation view of the compiled schedule */
typedef struct fw_scheduled_node {
    fw_node_id id;
    uint32_t num_inputs, num_outputs;
    uint32_t in_buffer[FW_MAX_PORTS];
    uint8_t in_should_clear[FW_MAX_PORTS];
    uint32_t out_buffer[FW_MAX_PORTS];
} fw_scheduled_node;

/* ---- context + graph (context.rs:36, graph.rs:125-580) ---------------------------------- */
FW_EXPORT void FW_FN(graph_config_default)(fw_graph_config* cfg);                  /* graph.rs:98-107 */
FW_EXPORT fw_ctx* FW_FN(ctx_new)(const fw_graph_config* cfg);                      /* context.rs:36 */
FW_EXPORT void FW_FN(ctx_free)(fw_ctx* ctx);                                        /* Drop context.rs:236-242 */
FW_EXPORT const char* FW_FN(ctx_last_error)(fw_ctx* ctx);                           /* Display of the last error */
FW_EXPORT fw_node_id FW_FN(graph_in_node)(fw_ctx* ctx);                             /* graph.rs:189 */
FW_EXPORT fw_node_id FW_FN(graph_out_node)(fw_ctx* ctx);                            /* graph.rs:194 */
FW_EXPORT fw_node_id FW_FN(graph_add_node)(fw_ctx* ctx, uint32_t num_inputs, uint32_t num_outputs,
                                           const fw_node_desc* desc);               /* graph.rs:201 */
/* add_node with a user node (graph.rs:201: `node: impl Into<Box<dyn AudioNode>>`). The vtable is copied; `node` is owned by
 * the graph from here on. Returns FW_ID_DANGLING (and drops the node) on bad arguments. */
FW_EXPORT fw_node_id FW_FN(graph_add_custom_node)(fw_ctx* ctx, uint32_t num_inputs, uint32_t num_outputs,
                                                  const fw_node_vtable* vtable, void* node);
/* Ok(Vec<EdgeID>) => 0 and *n_removed edges written (up to cap); Err(()) => -1 */
FW_EXPORT int FW_FN(graph_remove_node)(fw_ctx* ctx, fw_node_id node, fw_edge_id* removed, uint32_t cap,
                                       uint32_t* n_removed);                        /* graph.rs:268 */
FW_EXPORT int FW_FN(graph_set_num_inputs)(fw_ctx* ctx, fw_node_id node, uint32_t n, fw_edge_id* removed,
                                          uint32_t cap, uint32_t* n_removed);       /* graph.rs:315 */
FW_EXPORT int FW_FN(graph_set_num_outputs)(fw_ctx* ctx, fw_node_id node, uint32_t n, fw_edge_id* removed,
                                           uint32_t cap, uint32_t* n_removed);      /* graph.rs:349 */
/* returns fw_add_edge_error; on error *err_node / *err_port carry the payload of the variant */
FW_EXPORT int FW_FN(graph_connect)(fw_ctx* ctx, fw_node_id src, uint32_t src_port, fw_node_id dst,
                                   uint32_t dst_port, int check_for_cycles, fw_edge_id* out_edge,
                                   fw_node_id* err_node, uint32_t* err_port);       /* graph.rs:396 */
FW_EXPORT int FW_FN(graph_disconnect)(fw_ctx* ctx, fw_node_id src, uint32_t src_port, fw_node_id dst,
                                      uint32_t dst_port);                           /* graph.rs:483 -> bool */
FW_EXPORT int FW_FN(graph_disconnect_by_edge_id)(fw_ctx* ctx, fw_edge_id edge);     /* graph.rs:507 -> bool */
FW_EXPORT int FW_FN(graph_edge)(fw_ctx* ctx, fw_edge_id edge, fw_edge_info* out);   /* graph.rs:527 -> Option */
FW_EXPORT int FW_FN(graph_node_info)(fw_ctx* ctx, fw_node_id node, fw_node_info* out); /* graph.rs:253 -> Option */
FW_EXPORT uint32_t FW_FN(graph_num_nodes)(fw_ctx* ctx);                             /* graph.rs:302 */
FW_EXPORT uint32_t FW_FN(graph_num_edges)(fw_ctx* ctx);                             /* graph.rs:307 */
FW_EXPORT uint32_t FW_FN(graph_nodes)(fw_ctx* ctx, fw_node_id* out, uint32_t cap);  /* graph.rs:302 (slot order) */
FW_EXPORT uint32_t FW_FN(graph_edges)(fw_ctx* ctx, fw_edge_id* out, uint32_t cap);  /* graph.rs:307 (slot order) */
FW_EXPORT int FW_FN(graph_cycle_detected)(fw_ctx* ctx);                             /* graph.rs:573 */
FW_EXPORT void FW_FN(graph_reset)(fw_ctx* ctx);                                     /* graph.rs:171 */
FW_EXPORT int FW_FN(graph_needs_compile)(fw_ctx* ctx);                              /* graph.rs:582 */

/* compile_internal (graph.rs:629): compile without activation; the schedule is kept for
 * inspection through schedule_*. Returns fw_compile_error. */
FW_EXPORT int FW_FN(graph_compile_internal)(fw_ctx* ctx, uint32_t max_block_frames);
FW_EXPORT uint32_t FW_FN(schedule_len)(fw_ctx* ctx);                                /* schedule.rs:167 */
FW_EXPORT uint32_t FW_FN(schedule_num_buffers)(fw_ctx* ctx);                        /* schedule.rs:171 */
FW_EXPORT int FW_FN(schedule_node)(fw_ctx* ctx, uint32_t i, fw_scheduled_node* out);

/* ---- isomorphic-voice detection (ours; SURVEY §8 f2) ------------------------------------------------------------------------
 * The reference runs ONE graph; a mixer of V identical voices is V copies of a sub-graph that meet in a tree of SumNodes in front of
 * graph_out (the 64-port limit, compiler.rs:202-203, is why it is a tree). graph_detect_voices recognises that shape in a flat graph
 * (num_voices == 1): a balanced pairwise tree of 2-port SumNodes (2C inputs -> C outputs, sum.rs:69-81; an unpaired last element of a
 * level passes a 1-port SumNode, the copy path sum.rs:58-65) over V sub-graphs that are disjoint, read their own slice
 * [v * voice_inputs, (v + 1) * voice_inputs) of graph_in, and are isomorphic: same node kinds, port counts, wiring and static
 * parameters (stages, delay length, IR, tables, threshold); gains, pans and coefficients may differ — they become the per-voice tables.
 * ctx_new_batched then builds the equivalent batched context: the voice graph once, num_voices = V, master_bus = 1 — the bus IS that
 * tree, so the result is bit-identical to running the flat graph. A graph that is simply one voice answers num_voices == 1.
 * Returns 0, or -1 with the reason in ctx_last_error (the flat graph still runs as it is, through the generic lowering). */
typedef struct fw_voice_template {
    uint32_t num_voices;          /* V */
    uint32_t num_template_nodes;  /* nodes of one voice (graph_in / graph_out and the tree excluded), in canonical order */
    uint32_t voice_inputs, voice_outputs;  /* channels per voice */
    uint32_t num_tree_nodes;      /* SumNodes that disappear into the master bus */
} fw_voice_template;
FW_EXPORT int FW_FN(graph_detect_voices)(fw_ctx* flat, fw_voice_template* out);
/* after a successful detection: the ids, in the flat graph, of template node `template_node` in voice 0 .. V-1; returns V */
FW_EXPORT uint32_t FW_FN(graph_voice_nodes)(fw_ctx* flat, uint32_t template_node, fw_node_id* out, uint32_t cap);
/* the batched context of the detected graph (not activated; the flat context stays untouched and shares its sample resources).
 * template_ids[i] (cap entries, may be NULL) = id of template node i in the new graph. NULL + ctx_last_error(flat) on failure. */
FW_EXPORT fw_ctx* FW_FN(ctx_new_batched)(fw_ctx* flat, int32_t device, uint32_t max_call_frames, fw_node_id* template_ids, uint32_t cap);
/* main-thread view of a node's parameter table (the reference's getters: volume.rs:24,36, sampler.rs:167,179): copies up to cap
 * floats, returns the table's length — num_voices entries ([voice][stage][5 | 6] for FW_PARAM_COEFFS); 0: the node has no such table */
typedef enum fw_param_table { FW_PARAM_PERCENT_VOLUME = 0, FW_PARAM_RAW_GAIN = 1, FW_PARAM_PAN = 2, FW_PARAM_GAIN_L = 3, FW_PARAM_GAIN_R = 4, FW_PARAM_COEFFS = 5 } fw_param_table;
FW_EXPORT uint32_t FW_FN(node_read_params)(fw_ctx* ctx, fw_node_id node, uint32_t which, float* out, uint32_t cap);

/* ---- node parameters (main-thread side; relaxed-atomic stores in the reference) --------
 * The reference's processor polls per block: it drains its message ring and loads the atomic parameters at the top of every
 * process_block (processor.rs:214, volume.rs:92, sampler.rs:331), so a host that calls once per block places every store at a
 * block boundary of its choice. A batched call (K blocks) keeps that control: set_event_block(b) stamps the parameter stores
 * and sampler / resampler messages that FOLLOW with block offset b, counted from the first block of the NEXT process_* call;
 * they take effect exactly there (b = 0, the default: at the start of that call — the reference's behaviour for K = 1). Offsets
 * beyond that call carry over to the following one. Graph edits (ctx_update -> new schedule) and Stop are picked up at the
 * start of a call and at every boundary the call is split at; to swap a schedule at a chosen block, split the call there, as
 * a device callback period would. No call in this section takes a lock or blocks. */
FW_EXPORT void FW_FN(ctx_set_event_block)(fw_ctx* ctx, uint32_t block);
FW_EXPORT int FW_FN(volume_set_percent_volume)(fw_ctx* ctx, fw_node_id node, uint32_t voice, float percent); /* volume.rs:28 */
FW_EXPORT int FW_FN(volume_set_percent_volumes)(fw_ctx* ctx, fw_node_id node, const float* percent, uint32_t n_voices);
FW_EXPORT int FW_FN(pan_set_pan)(fw_ctx* ctx, fw_node_id node, uint32_t voice, float pan);
FW_EXPORT int FW_FN(pan_set_pans)(fw_ctx* ctx, fw_node_id node, const float* pan, uint32_t n_voices);
FW_EXPORT int FW_FN(pan_set_gains)(fw_ctx* ctx, fw_node_id node, uint32_t voice, float gain_l, float gain_r);
/* coeffs = {b0, b1, b2, a1, a2} (a0-normalised) */
FW_EXPORT int FW_FN(biquad_set_coeffs)(fw_ctx* ctx, fw_node_id node, uint32_t voice, uint32_t stage, const float* coeffs5);
/* coeffs: [voice][stage][5] */
FW_EXPORT int FW_FN(biquad_set_all_coeffs)(fw_ctx* ctx, fw_node_id node, const float* coeffs, uint32_t n_voices, uint32_t n_stages);
/* RBJ cookbook design, f64 -> f32, host only. type: 0 lowpass 1 highpass 2 bandpass 3 notch 4 peaking 5 lowshelf 6 highshelf */
FW_EXPORT void FW_FN(biquad_design_rbj)(uint32_t type, double fc, double q, double gain_db, double sample_rate, float* coeffs5);

/* SVF (SURVEY §8 a11, spec ours — DESIGN.md): per stage coeffs6 = {a1, a2, a3, m0, m1, m2}; per channel and stage, with
 * state (ic1, ic2):  v3 = x - ic2;  v1 = a1*ic1 + a2*v3;  v2 = ic2 + (a2*ic1 + a3*v3);  ic1 = 2*v1 - ic1;  ic2 = 2*v2 - ic2;
 * y = m0*x + (m1*v1 + m2*v2)   — every product and sum a single rounded f32 operation, in this order. */
FW_EXPORT int FW_FN(svf_set_coeffs)(fw_ctx* ctx, fw_node_id node, uint32_t voice, uint32_t stage, const float* coeffs6);
FW_EXPORT int FW_FN(svf_set_all_coeffs)(fw_ctx* ctx, fw_node_id node, const float* coeffs, uint32_t n_voices, uint32_t n_stages);
/* Simper/Cytomic design in f64 -> f32, host only: g = tan(pi*fc/sr), k = 1/q.
 * type: 0 lowpass 1 bandpass 2 highpass 3 notch 4 peak 5 allpass */
FW_EXPORT void FW_FN(svf_design)(uint32_t type, double fc, double q, double sample_rate, float* coeffs6);

/* Polyphase resampler (SURVEY §8 a13, spec ours — DESIGN.md). Per voice: a Q32.32 position `pos` and step `step`;
 * output frame n of a call reads at p = pos + n*step:  i = p >> 32,  phase = (p & 0xffffffff) >> (32 - log2 P),
 * y = sum_{t=0}^{T-1} table[phase][t] * x[i + t - (T/2 - 1)]   (t ascending, separate f32 multiply and add),
 * x = 0 outside [0, frames) or, with `loop`, indices taken modulo frames. After the call pos += frames_in_call * step.
 * Channel mapping as in the SamplerNode. Not playing / no resource => cleared and flagged. */
FW_EXPORT int FW_FN(resampler_set)(fw_ctx* ctx, fw_node_id node, uint32_t voice, uint32_t resource, uint64_t step_q32,
                                   int playing, int loop);
FW_EXPORT int FW_FN(resampler_seek)(fw_ctx* ctx, fw_node_id node, uint32_t voice, uint64_t pos_frames); /* next call starts here */
/* h[p][t] = cutoff * sinc(cutoff * (t - (T/2 - 1) - p/P)) * kaiser(beta), f64 -> f32; host only */
FW_EXPORT void FW_FN(resampler_design)(uint32_t phases, uint32_t taps, double cutoff, double beta, float* table);

/* ---- sample resources + SamplerNode (sample_resource.rs, sampler.rs:46-233) ---------------
 * A resource is uploaded once ("Arc<...>": shared by any number of voices and nodes) and lives until ctx_free.
 * Returns a handle >= 1, or 0 on bad arguments. `data` holds channels * frames elements of the format's type. */
FW_EXPORT uint32_t FW_FN(sample_resource_create)(fw_ctx* ctx, uint32_t format, uint32_t channels, uint64_t frames,
                                                 const void* data);
/* Messages to the processor side (sampler.rs:21-28); `voice` may be FW_ALL_VOICES. They are drained at the first
 * block of the next process call, in order (sampler.rs:331-414). */
FW_EXPORT int FW_FN(sampler_set_sample)(fw_ctx* ctx, fw_node_id node, uint32_t voice, uint32_t resource,
                                        int stop_playback);                         /* sampler.rs:67 */
FW_EXPORT int FW_FN(sampler_play)(fw_ctx* ctx, fw_node_id node, uint32_t voice);    /* sampler.rs:82 */
FW_EXPORT int FW_FN(sampler_pause)(fw_ctx* ctx, fw_node_id node, uint32_t voice);   /* sampler.rs:101 */
FW_EXPORT int FW_FN(sampler_stop)(fw_ctx* ctx, fw_node_id node, uint32_t voice);    /* sampler.rs:120 */
FW_EXPORT int FW_FN(sampler_set_playhead)(fw_ctx* ctx, fw_node_id node, uint32_t voice, double playhead_secs); /* :139 */
/* mode: fw_loop_mode; RANGE_SECS needs round(start*sr) < round(end*sr) (the reference underflows otherwise) */
FW_EXPORT int FW_FN(sampler_set_loop_range)(fw_ctx* ctx, fw_node_id node, uint32_t voice, uint32_t mode,
                                            double start_secs, double end_secs);    /* sampler.rs:153 */
FW_EXPORT int FW_FN(sampler_set_percent_volume)(fw_ctx* ctx, fw_node_id node, uint32_t voice, float percent); /* :174 */
FW_EXPORT int FW_FN(sampler_is_playing)(fw_ctx* ctx, fw_node_id node, uint32_t voice); /* node-side flag, sampler.rs:163 */

/* ---- lifecycle (context.rs:46-211) ------------------------------------------------------- */
/* 0 => *out_processor set (Some); 1 => already active (None) */
FW_EXPORT int FW_FN(ctx_activate)(fw_ctx* ctx, uint32_t sample_rate, uint32_t num_stream_in_channels,
                                  uint32_t num_stream_out_channels, uint32_t max_block_frames, void* user_cx,
                                  fw_processor** out_processor);                    /* context.rs:46 */
FW_EXPORT int FW_FN(ctx_is_activated)(fw_ctx* ctx);                                 /* context.rs:85 */
FW_EXPORT int FW_FN(ctx_update)(fw_ctx* ctx, fw_update_status* out);                /* context.rs:93 */
/* Blocks like the reference (Stop message, then 2 ms polls up to 3 s) until the processor has
 * been dropped with processor_free on the stream side. Returns the user_cx or NULL. */
FW_EXPORT void* FW_FN(ctx_deactivate)(fw_ctx* ctx, int stream_is_running);          /* context.rs:162 */

/* ---- the hot path (processor.rs:61-248, schedule.rs:213-343) ---------------------------- */
/* num_in_channels / num_out_channels must equal the counts given to ctx_activate; they may differ from graph_in's port count G_in
 * and graph_out's port count G_out, as in the reference (schedule.rs:213-287, util.rs:44-147):
 *   S1 n_in < G_in:   graph_in ports >= n_in read +0.0 in every block; downstream they are live zeros, not silent (graph_in's
 *                     Dummy overwrites their flags, schedule.rs:338-341);
 *   S2 n_in > G_in:   input channels >= G_in are ignored;
 *   S3 n_out > G_out: output channels >= G_out are written +0.0 and never flagged in a silence mask; with the master bus and two or
 *                     more voices the bus's SumNodes then never see all inputs flagged, so the bus mask is 0 (sum.rs:52-56);
 *   S4 n_out < G_out: graph_out ports >= n_out are not read; silence masks cover the n_out channels.
 * The master bus mixes min(G_out, n_out) channels. process_interleaved interleaves a stereo pair as one (util.rs:123-147) only when
 * n_out == 2 and G_out >= 2 (processor.rs:122-133). */
FW_EXPORT int FW_FN(processor_process_interleaved)(fw_processor* p, const float* input, float* output,
                                                   uint32_t num_in_channels, uint32_t num_out_channels,
                                                   uint64_t frames, double stream_time_secs,
                                                   uint32_t stream_status);         /* processor.rs:61 */
/* planar host buffers; *out_silence_mask = graph_out silence mask of the last block (schedule.rs:267-276) */
FW_EXPORT int FW_FN(processor_process_planar)(fw_processor* p, const float* input, float* output,
                                              uint32_t num_in_channels, uint32_t num_out_channels, uint64_t frames,
                                              double stream_time_secs, uint32_t stream_status,
                                              uint64_t* out_silence_mask);
/* planar DEVICE buffers, asynchronous on the processor's stream (product only) */
FW_EXPORT int FW_FN(processor_process_planar_device)(fw_processor* p, const float* d_input, float* d_output,
                                                     uint32_t num_in_channels, uint32_t num_out_channels,
                                                     uint64_t frames, double stream_time_secs, uint32_t stream_status);
FW_EXPORT void FW_FN(processor_free)(fw_processor* p);                              /* Drop processor.rs:251 */

/* ---- pull-style stream backend (product only; replaces firewheel-cpal's DataCallback, crates/firewheel-cpal/src/lib.rs:378-449)
 * cpal calls the processor from its device callback; here a producer thread renders `period_frames` at a time, ahead of
 * the consumer, into a host ring of `ring_periods` periods, and the consumer PULLS interleaved frames. Like cpal (lib.rs:177)
 * the stream has no input channels: activate with num_in_channels = 0, and graph_in's ports read +0.0 (S1 above); a graph whose
 * graph_out has fewer ports than the device has channels plays on the first ones (S3). stream_time_secs handed to the graph is the sample clock (frames rendered / sample
 * rate). A pull that finds the ring empty zero-fills the rest, reports FW_STREAM_OUTPUT_UNDERFLOW, and the next rendered
 * period carries that flag in its stream_status (lib.rs:424-428). After DropProcessor pulls deliver silence (lib.rs:446-448).
 * Requires one output stream per context: num_voices == 1 or master_bus == 1. While a stream is open the processor must not
 * be driven through process_* by anyone else. */
typedef struct fw_stream fw_stream;
FW_EXPORT fw_stream* FW_FN(stream_open)(fw_processor* p, uint32_t num_out_channels, uint32_t sample_rate, uint32_t period_frames,
                                        uint32_t ring_periods);
/* returns the frames delivered (<= frames; the rest of `out` is zero-filled); *status gets fw_stream_status bits;
 * *stream_time_secs = frames delivered before this pull / sample_rate */
FW_EXPORT int64_t FW_FN(stream_pull)(fw_stream* s, float* out_interleaved, uint64_t frames, uint32_t* status, double* stream_time_secs);
FW_EXPORT uint64_t FW_FN(stream_frames_ready)(fw_stream* s);
FW_EXPORT void FW_FN(stream_close)(fw_stream* s);   /* joins the producer thread; the processor stays alive */

/* ---- device plumbing for drivers and benchmarks (product only; oracle returns errors) --- */
FW_EXPORT int FW_FN(device_count)(void);
FW_EXPORT const char* FW_FN(last_device_error)(void);
FW_EXPORT void* FW_FN(dev_malloc)(int device, uint64_t bytes);
FW_EXPORT void FW_FN(dev_free)(int device, void* p);
FW_EXPORT void* FW_FN(host_alloc_pinned)(uint64_t bytes);
FW_EXPORT void FW_FN(host_free_pinned)(void* p);
FW_EXPORT int FW_FN(processor_h2d)(fw_processor* p, void* dst, const void* src, uint64_t bytes);  /* async on the stream */
FW_EXPORT int FW_FN(processor_d2h)(fw_processor* p, void* dst, const void* src, uint64_t bytes);
FW_EXPORT int FW_FN(processor_sync)(fw_processor* p);
/* CUDA events on the processor's stream: record slot 0/1, elapsed in ms */
FW_EXPORT int FW_FN(processor_event_record)(fw_processor* p, int slot);
FW_EXPORT float FW_FN(processor_event_elapsed_ms)(fw_processor* p, int slot_start, int slot_stop);
FW_EXPORT uint64_t FW_FN(processor_kernel_launches)(fw_processor* p); /* kernels launched so far */
FW_EXPORT uint64_t FW_FN(processor_graph_replays)(fw_processor* p);   /* chunks replayed from a captured CUDA graph so far */
/* Per-kernel-class device timing with CUDA events on the launching stream.
 * classes: 0 control, 1 fused chain (+bus), 2 bus combine, 3 temporal (biquad/delay/reverb). */
FW_EXPORT int FW_FN(processor_profile)(fw_processor* p, int enable);
FW_EXPORT int FW_FN(processor_profile_read)(fw_processor* p, double* ms_by_class4, uint64_t* launches_by_class4);
FW_EXPORT int FW_FN(processor_l2_flush)(fw_processor* p);             /* writes a >L2 scratch buffer */

/* ---- multi-GPU master bus (voices sharded by rank; SURVEY §8e) --------------------------- */
FW_EXPORT int FW_FN(comm_unique_id)(uint8_t* id128);                  /* ncclGetUniqueId */
FW_EXPORT int FW_FN(processor_comm_init)(fw_processor* p, int rank, int world_size, const uint8_t* id128);
/* host-buffer all-gather over that communicator (recv holds world_size * bytes): barriers, max-over-ranks timing and
 * cross-rank result checks of a torch-free driver; world_size == 1 copies. Not on the audio path. */
FW_EXPORT int FW_FN(processor_comm_allgather)(fw_processor* p, const void* send, void* recv, uint64_t bytes);

#ifdef __cplusplus
}
#endif
#endif /* FW_B200_H */
