/*
 * kvbm_physical.h -- C ABI of libkvbm_physical.so: the host half of the KV transfer path.
 *
 * It restates, in C++ behind plain-C entry points, what Dynamo's Rust crate lib/kvbm-physical does for
 * this path (no Rust toolchain exists in the build image; see INTEGRATION.md for the Rust `extern "C"`
 * block a maintainer would add):
 *
 *   LayoutConfig + validation            lib/kvbm-physical/src/layout/config.rs:14-56,165-180
 *   FullyContiguous / LayerSeparate      layout/fully_contiguous.rs:141-185, layout/layer_separate.rs:155-210
 *   Layout::memory_region                layout/mod.rs:73-78
 *   validate_block_transfer              transfer/validation.rs:55-225
 *   select_strategy / direct strategy    transfer/strategy.rs:78-108,138-210
 *   TransferOptions                      transfer/options.rs:27-81
 *   TransferManager::{register_layout, export_metadata, import_metadata, execute_transfer}
 *                                        manager/mod.rs:101,112,130,227
 *   TransferCompleteNotification         transfer/context.rs:438-470 (event -> 1 ms poller) -- replaced by an
 *                                        in-band completion flag the kernel writes to pinned host memory
 *   layer-wise onboard                   lib/kvbm-engine/src/worker/physical.rs:277-346
 *   CollectiveOps::broadcast             lib/kvbm-engine/src/collectives/mod.rs:75-106 (ncclBcast per region)
 *                                        -- replaced by one replicate launch over NVLink peer mappings
 *
 * Threading: a kvbm_transfer_manager may be used from any number of threads concurrently (the reference is called from
 * arbitrary tokio workers); checked under ThreadSanitizer by tests/c/race_check.cpp.
 * Error style: every call returns KVBM_OK (0) or an error code; kvbm_last_error() gives the thread's last
 * message (house style of lib/bindings/c/src/lib.rs:74-78: OK=0, ERR!=0).  Nothing aborts or throws.
 */
#ifndef KVBM_PHYSICAL_H
#define KVBM_PHYSICAL_H

#include <stddef.h>
#include <stdint.h>

#include "kvbm_kernels.h"

#ifdef __cplusplus
extern "C" {
#endif

enum {
  KVBM_OK = 0,
  KVBM_ERR = 1,                 /* generic */
  KVBM_ERR_CONFIG = 2,          /* LayoutConfig validation failed / memory too small */
  KVBM_ERR_RANGE = 3,           /* block / layer / outer id out of range */
  KVBM_ERR_LENGTH_MISMATCH = 4, /* BlockValidationError::LengthMismatch */
  KVBM_ERR_DUPLICATE_DST = 5,   /* BlockValidationError::DuplicateDestinationBlocks */
  KVBM_ERR_OVERLAP = 6,         /* BlockValidationError::OverlappingBlocks */
  KVBM_ERR_INCOMPATIBLE = 7,    /* layer count / outer dim / region size mismatch */
  KVBM_ERR_UNSUPPORTED = 8,     /* strategy this library does not implement (NIXL, disk, System<->Device) */
  KVBM_ERR_CUDA = 9,            /* a CUDA call failed (message carries the cudaError_t) */
  KVBM_ERR_HANDLE = 10,         /* unknown layout handle / notification */
  KVBM_ERR_TIMEOUT = 11,
  KVBM_ERR_VERSION = 12,        /* metadata blob version mismatch (layout/serialize.rs version check) */
};

/* dynamo_memory::StorageKind (lib/memory/src/lib.rs) */
enum { KVBM_STORAGE_SYSTEM = 0, KVBM_STORAGE_PINNED = 1, KVBM_STORAGE_DEVICE = 2, KVBM_STORAGE_DISK = 3 };
/* BlockDimension (layout/config.rs:151-163) */
enum { KVBM_BLOCK_IS_FIRST_DIM = 0, KVBM_BLOCK_IS_SECOND_DIM = 1 };
/* TransferStrategy (transfer/strategy.rs:20-58) */
enum {
  KVBM_STRATEGY_MEMCPY = 0,
  KVBM_STRATEGY_CUDA_ASYNC_H2D = 1,
  KVBM_STRATEGY_CUDA_ASYNC_D2H = 2,
  KVBM_STRATEGY_CUDA_ASYNC_D2D = 3,
  KVBM_STRATEGY_NIXL_READ = 4,
  KVBM_STRATEGY_NIXL_WRITE = 5,
  KVBM_STRATEGY_NIXL_READ_FLIPPED = 6,
  KVBM_STRATEGY_INVALID = 7,
};

typedef struct kvbm_layout_config {
  size_t num_blocks;
  size_t num_layers;
  size_t outer_dim;         /* 1 or 2 */
  size_t page_size;
  size_t inner_dim;
  size_t alignment;         /* power of two; 0 is read as 1 (the builder default) */
  size_t dtype_width_bytes; /* 2,4,8 as the reference; 1 accepted only with allow_fp8 */
  size_t num_heads;         /* 0 = None */
  int allow_fp8;            /* extension: fp8 KV pools (dtype_width_bytes == 1) */
} kvbm_layout_config;

/* A transfer plan as select_strategy returns it (transfer/strategy.rs:60-76). */
typedef struct kvbm_transfer_plan {
  int two_hop;          /* 0 = Direct(first) */
  int first;            /* KVBM_STRATEGY_* */
  int bounce_location;  /* KVBM_STORAGE_* (two-hop only) */
  int second;           /* two-hop only */
} kvbm_transfer_plan;

typedef struct kvbm_transfer_capabilities {
  int allow_gds;
  int allow_gpu_rdma;
} kvbm_transfer_capabilities;

/* TransferOptions (transfer/options.rs:27-81) + the cast / streaming extensions. */
typedef struct kvbm_transfer_options {
  int has_layer_range;
  size_t layer_begin, layer_end;
  cudaStream_t cuda_stream;     /* non-NULL: caller manages sync, notification is already complete */
  int use_caller_stream;        /* set when cuda_stream is meaningful (NULL is the legacy default stream) */
  int cast_mode;                /* KVBM_CAST_* */
  int max_ctas;                 /* 0 = whole GPU; else cap so attention keeps its SMs */
  const uint32_t* layer_ready_flags; /* nullable: device flags released by the producer (attention) per layer */
  uint32_t* layer_done_flags;        /* nullable: device-visible flags on the destination, set per layer */
  uint32_t epoch;
  int gate_timeout_ms;               /* 0 = 10 s; see kvbm_paged_copy_opts.gate_timeout_ms */
  int multicast;                     /* non-zero: the destination layout is registered over a kvbm_mc_group_map() range */
  uint32_t* done_flag;               /* nullable: word in the DESTINATION GPU's memory that receives `epoch` once every byte of
                                        the transfer has landed -- the role of TransferOptions::nixl_write_notification
                                        (options.rs:36-43: "delivered to the remote node after the RDMA write completes") */
  /* BounceBuffer (options.rs:45-51): a registered layout + the blocks of it a two-hop transfer may stage through */
  uint64_t bounce_layout;            /* kvbm_layout_handle; 0 = none */
  const size_t* bounce_block_ids;
  size_t num_bounce_blocks;
  int src_kv_layout, dst_kv_layout;  /* KvBlockLayout overrides, KVBM_KV_* (options.rs:63-80): 0 = the layout's own.  A pair that
                                        needs a transformation is EXECUTED as one permuting launch (the reference rejects it,
                                        transfer/mod.rs:128-147): see kvbm_select_transform_kernel */
  int gate_mode;                     /* see kvbm_paged_copy_opts.gate_mode */
  /* fan-out only: per-destination signals (arrays of num_dsts pointers, entries may be NULL).  When set they replace
   * done_flag / layer_done_flags, which only reach destination 0.  With `multicast` they name the flags of every receiver of
   * the one multicast write -- what a staged broadcast needs (disagg.StagedBroadcast). */
  uint32_t* const* per_dst_done_flags;
  uint32_t* const* per_dst_layer_done_flags;
  /* head window (tensor-parallel re-shard): heads [src_head_begin, src_head_begin + head_count) of each source block land as
   * heads [dst_head_begin, dst_head_begin + head_count) of its destination block; every other destination byte keeps its
   * value.  head_count 0 = every head (no window).  The two layouts may have different num_heads; see
   * kvbm_manager_execute_transfer for the rules. */
  size_t src_head_begin, dst_head_begin, head_count;
  /* fp8 KV-cache scales: with a cast_mode, cast_scales[l * outer_dim + o] is the dequantisation scale of the FP8 side for layer
   * l (absolute) and outer index o, applied by every cast launch (kvbm_paged_copy_opts.cast_scales has the formulas).  NULL =
   * unscaled.  num_cast_scales must be at least num_layers * outer_dim (KVBM_ERR_RANGE); scales without a cast_mode and a pointer
   * the manager's device cannot read (anything but its own device memory or pinned host memory mapped into it) are KVBM_ERR.
   * All three are rejected before any launch.  A gather applies one array to every source. */
  const float* cast_scales;
  size_t num_cast_scales;
} kvbm_transfer_options;

typedef struct kvbm_transfer_manager kvbm_transfer_manager;
typedef uint64_t kvbm_layout_handle;   /* (worker_id << 16) | layout_id, cf. manager/handle.rs:16-50 */
typedef uint64_t kvbm_notification;    /* 0 = already complete */

const char* kvbm_last_error(void);

/* ---- pure host logic (no GPU needed) ---- */
int kvbm_layout_config_validate(const kvbm_layout_config* cfg);
size_t kvbm_layout_required_bytes(const kvbm_layout_config* cfg);   /* config.rs:64-71 */
size_t kvbm_layout_bytes_per_block(const kvbm_layout_config* cfg);  /* config.rs:76-82 */
/* select_direct_strategy (strategy.rs:138-210).  Device ids are ignored exactly as strategy.rs:168 does. */
int kvbm_select_direct_strategy(int src_kind, int dst_kind, const kvbm_transfer_capabilities* caps,
                                kvbm_transfer_plan* out);
/* The same with select_direct_strategy's `dst_is_remote` argument (strategy.rs:138-150, select_remote_strategy :213-243): a local
 * source to another agent's memory is NixlWrite, staged through Pinned for Device (without GPU RDMA) and Disk. */
int kvbm_select_direct_strategy_remote(int src_kind, int dst_kind, int dst_is_remote, const kvbm_transfer_capabilities* caps,
                                       kvbm_transfer_plan* out);
/* select_strategy (strategy.rs:78-108) with select_remote_strategy_v2 (:245-281): both local = the table above; exactly one
 * side local = NixlWrite (push) or NixlReadFlipped (pull) -- executed here as the push / pull launch over the IPC-mapped pool;
 * both remote, Disk, or a Device side without allow_gpu_rdma = the reference's errors. */
int kvbm_select_strategy(int src_kind, int src_is_local, int dst_kind, int dst_is_local, const kvbm_transfer_capabilities* caps,
                         kvbm_transfer_plan* out);
/* validate_block_transfer, debug flavour (validation.rs:168-225). */
int kvbm_validate_block_transfer(const size_t* src_ids, size_t n_src, const size_t* dst_ids, size_t n_dst,
                                 size_t src_num_blocks, size_t dst_num_blocks, int same_layout);

/* One entry of a tensor-parallel re-shard plan: heads [src_head_begin, src_head_begin + head_count) of source rank src_rank's
 * blocks are heads [dst_head_begin, dst_head_begin + head_count) of the decode rank's blocks (rank-local head indices). */
typedef struct kvbm_head_window {
  size_t src_rank, src_head_begin, dst_head_begin, head_count;
} kvbm_head_window;
/* Which source rank supplies which heads of decode rank dst_rank when num_kv_heads KV heads are sharded over src_tp ranks on
 * the source side and dst_tp on the destination side.  Ownership follows vLLM: with tp ranks and H heads, rank r holds heads
 * [r*H/tp, r*H/tp + max(1, H/tp)); when tp > H each head is replicated over tp/H ranks and the plan reads replica
 * dst_rank % (tp/H), so concurrent pulls of different decode ranks spread over the source GPUs.  Windows come out in ascending
 * destination head order; adjacent heads from the same source rank are merged.  H % tp or tp % H must be 0 on both sides
 * (else KVBM_ERR_CONFIG, as is a zero argument); dst_rank >= dst_tp is KVBM_ERR_RANGE.  *n_out receives the number of
 * windows; out == NULL only counts, a cap below the count is KVBM_ERR.  Pure host logic. */
int kvbm_tp_reshard_plan(size_t num_kv_heads, size_t src_tp, size_t dst_tp, size_t dst_rank, kvbm_head_window* out, size_t cap,
                         size_t* n_out);

/* One entry of a pipeline- and tensor-parallel re-shard plan: heads [src_head_begin, +head_count) of layers [src_layer_begin,
 * +layer_count) of source rank src_rank's blocks are heads [dst_head_begin, +head_count) of layers [dst_layer_begin,
 * +layer_count) of the decode rank's blocks.  Layers are stage-local on each side (layer 0 of a pool is the first layer of its
 * pipeline stage), heads rank-local. */
typedef struct kvbm_shard_window {
  size_t src_rank, src_layer_begin, dst_layer_begin, layer_count, src_head_begin, dst_head_begin, head_count;
} kvbm_shard_window;
/* Which source rank supplies which layers and heads of decode rank dst_rank when num_layers layers of num_kv_heads KV heads are
 * split over src_pp pipeline stages of src_tp ranks on the source side and dst_pp x dst_tp on the destination side.  Ranks are
 * numbered pp_rank * tp + tp_rank on both sides.  src_stage_layers / dst_stage_layers: each stage's layer count ([pp] entries,
 * ascending stages); NULL splits evenly, which needs num_layers % pp == 0.  For each source stage that shares layers with the
 * decode rank's stage, the plan holds kvbm_tp_reshard_plan's head windows of that pair of TP degrees (its ownership and replica
 * rule, for tp rank dst_rank % dst_tp) over the shared layers, in ascending destination layer, then destination head order.
 * With src_pp = dst_pp = 1 it is kvbm_tp_reshard_plan's plan over every layer.  Errors: KVBM_ERR a null n_out or a cap below the
 * count (out == NULL only counts); KVBM_ERR_CONFIG a zero argument, num_layers % pp != 0 with a NULL partition, a partition with
 * a zero stage or that does not sum to num_layers, and kvbm_tp_reshard_plan's head rule; KVBM_ERR_RANGE dst_rank >= dst_pp *
 * dst_tp.  Pure host logic. */
int kvbm_tp_pp_reshard_plan(size_t num_kv_heads, size_t num_layers, size_t src_tp, size_t src_pp, const size_t* src_stage_layers,
                            size_t dst_tp, size_t dst_pp, const size_t* dst_stage_layers, size_t dst_rank, kvbm_shard_window* out,
                            size_t cap, size_t* n_out);

/* One entry of a scatter plan: heads [src_head_begin, +head_count) of layers [src_layer_begin, +layer_count) of the prefill rank's
 * blocks are heads [dst_head_begin, +head_count) of layers [dst_layer_begin, +layer_count) of decode rank dst_rank's blocks
 * (stage-local layers, rank-local heads, as kvbm_shard_window). */
typedef struct kvbm_scatter_window {
  size_t dst_rank, src_layer_begin, dst_layer_begin, layer_count, src_head_begin, dst_head_begin, head_count;
} kvbm_scatter_window;
/* The push side of kvbm_tp_pp_reshard_plan: which layers and heads of prefill rank src_rank go to which decode rank.  Defined as
 * the inverse of the gather plans: exactly the windows with that src_rank of kvbm_tp_pp_reshard_plan over every decode rank, each
 * tagged with its decode rank, in ascending (dst_rank, destination layer, destination head) order.  Replicated heads follow the
 * gather plan's replica rule (replica dst_rank % replicas), so the push and pull plans of one group move the same bytes.  The
 * arguments, errors and count / cap convention are kvbm_tp_pp_reshard_plan's, with KVBM_ERR_RANGE for src_rank >= src_pp * src_tp
 * in place of its dst_rank rule.  Pure host logic. */
int kvbm_tp_pp_scatter_plan(size_t num_kv_heads, size_t num_layers, size_t src_tp, size_t src_pp, const size_t* src_stage_layers,
                            size_t dst_tp, size_t dst_pp, const size_t* dst_stage_layers, size_t src_rank, kvbm_scatter_window* out,
                            size_t cap, size_t* n_out);

/* ---- TransferManager ---- */
/* cuda_device_id < 0: host-only manager (Memcpy strategy only; every CUDA strategy returns KVBM_ERR_CUDA). */
int kvbm_manager_create(int cuda_device_id, uint64_t worker_id, kvbm_transfer_manager** out);
void kvbm_manager_destroy(kvbm_transfer_manager* m);

/* register_layout over caller-owned memory (the engine's KV tensors).  device_id is where the memory lives
 * (may differ from the manager's device: a peer GPU reachable over NVLink). */
int kvbm_manager_register_fully_contiguous(kvbm_transfer_manager* m, const kvbm_layout_config* cfg, void* base,
                                           size_t size, int storage_kind, int device_id,
                                           kvbm_layout_handle* out);
int kvbm_manager_register_layer_separate(kvbm_transfer_manager* m, const kvbm_layout_config* cfg,
                                         void* const* layer_bases, const size_t* layer_sizes, int block_dim,
                                         int storage_kind, int device_id, kvbm_layout_handle* out);
int kvbm_manager_unregister(kvbm_transfer_manager* m, kvbm_layout_handle h);
int kvbm_layout_memory_region(kvbm_transfer_manager* m, kvbm_layout_handle h, size_t block, size_t layer,
                              size_t outer, uintptr_t* addr, size_t* size);
int kvbm_layout_is_fully_contiguous(kvbm_transfer_manager* m, kvbm_layout_handle h);

/* Enable NVLink peer mappings from the manager's device to `peer_device` (same process). */
int kvbm_manager_enable_peer_access(kvbm_transfer_manager* m, int peer_device);

/* export_metadata / import_metadata (manager/mod.rs:112,130): a self-describing blob carrying the layout
 * geometry and, for Device storage, one CUDA IPC handle per allocation, so another PROCESS on the same
 * NVSwitch domain can map the pool and have the transfer kernel store into it directly.
 * kvbm_manager_export_metadata with buf == NULL returns the needed size in *len. */
int kvbm_manager_export_metadata(kvbm_transfer_manager* m, kvbm_layout_handle h, void* buf, size_t cap,
                                 size_t* len);
int kvbm_manager_import_metadata(kvbm_transfer_manager* m, const void* buf, size_t len, kvbm_layout_handle* out);
/* The same for HOST pools (System / Pinned) of another process that this process has mapped itself -- shared memory, a file
 * mapping, memory shared across fork: local_bases[i] is this process's address of the layout's i-th allocation (1 for fully
 * contiguous, num_layers for layer-separate).  Without it such a layout is imported as a descriptor only (no transfer may touch
 * it).  The CPU twin of the CUDA-IPC mapping: BASELINE configs[0]'s two-process memcpy hand-off is a one-sided push too. */
int kvbm_manager_import_metadata_mapped(kvbm_transfer_manager* m, const void* buf, size_t len, const void* const* local_bases,
                                        size_t num_local_bases, kvbm_layout_handle* out);

/* The reference's own wire formats for the handshake (SURVEY.md 8 f3):
 *   kvbm_manager_export_serialized_layout / import_serialized_layout = TransferManager::export_metadata / import_metadata
 *   (manager/mod.rs:112,130): ONE blob for every local host/device layout, encoded exactly as SerializedLayout::pack
 *   (manager/metadata.rs:120-134: bincode 2 standard config over RdmaLayoutDescriptors).  Its `nixl_metadata` byte
 *   field carries this library's CUDA-IPC transport records instead of a NIXL agent's metadata; a second import of
 *   the same (agent, worker_id) fails like the reference ("Remote worker already loaded").  import with out == NULL
 *   returns the number of layouts in *n_out.
 *   kvbm_layout_descriptor_json / kvbm_manager_import_descriptor_json = LayoutDescriptor::to_json / from_json +
 *   PhysicalLayout::from_descriptor (layout/serialize.rs:96-137, layout/physical.rs:203-262); JSON-imported layouts
 *   keep the addresses as written (same address space).  Handles on the wire are the reference's u128
 *   (worker_id | layout_id << 64, manager/handle.rs:16-24); this ABI's 64-bit handle is (worker_id << 16) | layout_id. */
int kvbm_manager_export_serialized_layout(kvbm_transfer_manager* m, void* buf, size_t cap, size_t* len);
int kvbm_manager_import_serialized_layout(kvbm_transfer_manager* m, const void* buf, size_t len, kvbm_layout_handle* out,
                                          size_t cap, size_t* n_out);
int kvbm_layout_descriptor_json(kvbm_transfer_manager* m, kvbm_layout_handle h, char* buf, size_t cap, size_t* len);
int kvbm_manager_import_descriptor_json(kvbm_transfer_manager* m, const char* json, size_t len, kvbm_layout_handle* out);

/* select_strategy for two registered layouts (local = registered or imported in-process; remote = imported from another process) */
int kvbm_manager_select_strategy(kvbm_transfer_manager* m, kvbm_layout_handle src, kvbm_layout_handle dst, kvbm_transfer_plan* out);

/* TransformKernel (transfer/executor/mod.rs:27-41) as select_transform_kernel (:46-100) returns it. */
enum {
  KVBM_TRANSFORM_NONE = 0,
  KVBM_TRANSFORM_BLOCK_TO_UNIVERSAL = 1,
  KVBM_TRANSFORM_UNIVERSAL_TO_BLOCK = 2,
  KVBM_TRANSFORM_OPERATIONAL_TRANSPOSE = 3,
  KVBM_TRANSFORM_UNSUPPORTED = 4,
  KVBM_TRANSFORM_UNIVERSAL_TO_UNIVERSAL = 5, /* extension: UniversalTP <-> UniversalPP, a TODO in the reference (:87-91);
                                                never returned by kvbm_select_transform_kernel, but executed by transfers */
};
int kvbm_select_transform_kernel(int src_kv_layout, int dst_kv_layout);       /* pure; KVBM_KV_* in, KVBM_TRANSFORM_* out */
int kvbm_kv_layout_requires_transform(int a, int b);                          /* kv_block_layout.rs:107-119 */
/* The format of one block of a registered layout (FullyContiguousLayoutBuilder::kv_block_layout, fully_contiguous.rs:83-88;
 * LayerSeparateLayoutBuilder::inner_shape, layer_separate.rs:91-101).  Needs num_heads in the config; universal formats need
 * a fully contiguous layout.  Travels with export_metadata / the SerializedLayout. */
int kvbm_manager_set_kv_block_layout(kvbm_transfer_manager* m, kvbm_layout_handle h, int kv_layout);
int kvbm_manager_kv_block_layout(kvbm_transfer_manager* m, kvbm_layout_handle h);  /* KVBM_KV_*, -1 = unknown handle */

/* TransferCapabilities (transfer/strategy.rs:245-278).  Default {allow_gds 0, allow_gpu_rdma 1}.  With allow_gpu_rdma = 0 a
 * Device -> Device transfer between different GPUs follows the reference's TwoHop plan (strategy.rs:222-233):
 * CudaAsyncD2H into the bounce buffer named in the options (Pinned), then CudaAsyncH2D into the destination; the bounce blocks
 * are split into two groups and the hops of consecutive chunks overlap (executor/mod.rs:357-416,477-571).  Without a bounce
 * buffer such a transfer fails with "Two-hop transfers require a bounce buffer." as in the reference. */
int kvbm_manager_set_capabilities(kvbm_transfer_manager* m, const kvbm_transfer_capabilities* caps);

/* execute_transfer (manager/mod.rs:227-303).  ids are host arrays, consumed before return. */
int kvbm_manager_execute_transfer(kvbm_transfer_manager* m, kvbm_layout_handle src, const size_t* src_ids,
                                  kvbm_layout_handle dst, const size_t* dst_ids, size_t n,
                                  const kvbm_transfer_options* opts, kvbm_notification* out);

/* 1 -> N in ONE launch.  src_ids[d] == src_ids[0] for all d (same pointer or same contents flag
 * `replicate`) reads HBM once and stores N times: the replacement of CollectiveOps::broadcast. */
int kvbm_manager_execute_fanout(kvbm_transfer_manager* m, kvbm_layout_handle src, int num_dsts,
                                const kvbm_layout_handle* dsts, const size_t* const* src_ids,
                                const size_t* const* dst_ids, size_t n, int replicate,
                                const kvbm_transfer_options* opts, kvbm_notification* out);

/* N -> 1 in ONE launch: a decode rank assembles its blocks from several source pools (a TP re-shard plan,
 * kvbm_tp_reshard_plan).  windows[j].src_rank indexes srcs / src_ids, so a plan can be passed as it is; a source may appear in
 * several windows.  Heads [src_head_begin, +head_count) of block src_ids[src_rank][i] land as heads [dst_head_begin,
 * +head_count) of block dst_ids[i]; every other destination byte keeps its value.  Each (source, destination) pair must pass
 * what a windowed kvbm_manager_execute_transfer checks and is rejected with the same codes and texts (formats, head rows,
 * casts, contiguity, alignment, block ids, layer range, layer streaming / multicast / fan-out flags, Two-hop and Memcpy
 * strategies, both remote); all sources must select the same CUDA strategy.  Also: at most KVBM_GATHER_MAX_SOURCES (16)
 * windows (KVBM_ERR_UNSUPPORTED), src_rank >= num_srcs or an empty window (KVBM_ERR_RANGE), windows overlapping in the
 * destination (KVBM_ERR_OVERLAP), opts->head_count != 0 (KVBM_ERR).  One H2D upload of the (num_srcs + 1) * n ids, one
 * kvbm_kernels_paged_permute_gather launch, one signal launch: opts->done_flag and the notification complete once, after
 * every window's bytes landed.  bytes_moved counts each window's destination bytes. */
int kvbm_manager_execute_gather(kvbm_transfer_manager* m, size_t num_srcs, const kvbm_layout_handle* srcs,
                                const size_t* const* src_ids, kvbm_layout_handle dst, const size_t* dst_ids, size_t n,
                                const kvbm_head_window* windows, size_t num_windows, const kvbm_transfer_options* opts,
                                kvbm_notification* out);

/* Re-paging hand-off between engines with different page sizes, over any token range: tokens [token_begin, token_end) of one
 * sequence move from src's block table to dst's, each layout with its own page_size (one must divide the other; equal sizes are
 * a token-range copy).  Token p sits in slot p % P of block table[p / P] on a side of page P, so src_ids holds
 * src_table[token_begin / Ps .. ceil(token_end / Ps)) (n_src ids) and dst_ids dst_table[token_begin / Pd .. ceil(token_end / Pd))
 * (n_dst ids).  Every layer of the options' layer range, outer index and head of those tokens is re-ordered between the two
 * formats and cast as opts->cast_mode / cast_scales say; every other destination byte keeps its value, including the slots
 * of the first and last destination blocks outside the range.  Honoured options: the layer range, cast_mode, cast_scales /
 * num_cast_scales, src_kv_layout / dst_kv_layout, done_flag / epoch and the caller stream.  Errors, first one wins:
 * KVBM_ERR_HANDLE unknown handle; KVBM_ERR_UNSUPPORTED an unmapped host descriptor, both sides remote, a head window, layer
 * streaming / per-destination flags / multicast / a bounce buffer in the options, or a format that is not named (1..4);
 * KVBM_ERR_CONFIG num_heads missing or not dividing inner_dim; KVBM_ERR_INCOMPATIBLE layer count, outer dim, head row, cast
 * dtype, num_heads or dtype mismatch, pages that do not divide, and the permuting path's row, contiguity and alignment rules
 * (KVBM_ERR_UNSUPPORTED for rows and alignment, as execute_transfer); KVBM_ERR_RANGE token_begin > token_end or token_end
 * past 2^31, a layer range past num_layers, too few cast scales; KVBM_ERR_LENGTH_MISMATCH n_src / n_dst other than the counts
 * the range implies; KVBM_ERR_DUPLICATE_DST / KVBM_ERR_OVERLAP / KVBM_ERR_RANGE for ids as kvbm_validate_block_transfer;
 * an empty token or layer range then returns KVBM_OK with nothing launched; KVBM_ERR_UNSUPPORTED a strategy other than a
 * direct CUDA one (Memcpy, two-hop, NIXL); KVBM_ERR_CUDA a host-only manager.  One upload of both id lists, one
 * kvbm_kernels_paged_repage launch; bytes_moved counts tokens * layers * outer_dim * num_heads * the destination row. */
int kvbm_manager_execute_repage(kvbm_transfer_manager* m, kvbm_layout_handle src, const size_t* src_ids, size_t n_src,
                                kvbm_layout_handle dst, const size_t* dst_ids, size_t n_dst, size_t token_begin, size_t token_end,
                                const kvbm_transfer_options* opts, kvbm_notification* out);

/* A TP re-shard's assembly across engines with different page sizes (prefill pages of Ps tokens at one TP degree, decode pages
 * of Pd at another), as ONE hand-off: kvbm_manager_execute_gather's windows over kvbm_manager_execute_repage's token range.  For
 * window w, head w.src_head_begin + j of source w.src_rank lands as destination head w.dst_head_begin + j (j < w.head_count), at
 * every token of [token_begin, token_end), every layer of the options' layer range and every outer index, re-ordered and cast as
 * execute_repage would.  src_ids[s] holds source s's table[token_begin / Ps .. ceil(token_end / Ps)) (n_src ids each), dst_ids
 * the destination's table[token_begin / Pd .. ceil(token_end / Pd)) (n_dst ids).  Every other destination byte keeps its value:
 * heads no window covers, and the slots of the first and last destination blocks outside the range.  windows are
 * kvbm_head_windows, so a kvbm_tp_reshard_plan passes as it is.  Honoured options: execute_repage's (src_kv_layout applies to
 * every source).  Errors, first one wins: execute_gather's window checks (KVBM_ERR no source or window, or options.head_count;
 * KVBM_ERR_UNSUPPORTED more than KVBM_GATHER_MAX_SOURCES windows; KVBM_ERR_RANGE a window naming no source or with no heads;
 * KVBM_ERR_OVERLAP two windows on one destination head); KVBM_ERR_HANDLE; then for each window's source, execute_repage's checks
 * of its pair with the destination (num_heads may differ), the window inside both sides' heads (KVBM_ERR_RANGE) and
 * KVBM_ERR_INCOMPATIBLE a page size other than the first source's; execute_repage's token range, layer range, cast scales and
 * id counts (KVBM_ERR_LENGTH_MISMATCH n_src / n_dst other than the range implies for Ps / Pd); the ids of each window's source
 * against the destination's, as execute_repage; an empty token or layer range then returns KVBM_OK with nothing launched;
 * KVBM_ERR_UNSUPPORTED a strategy other than a direct CUDA one, or sources with different ones; KVBM_ERR_CUDA a host-only
 * manager.  One upload of num_srcs * n_src + n_dst ids, one kvbm_kernels_paged_repage_gather launch, one notification;
 * bytes_moved counts tokens * layers * outer_dim * covered heads * the destination row. */
int kvbm_manager_execute_repage_gather(kvbm_transfer_manager* m, size_t num_srcs, const kvbm_layout_handle* srcs,
                                       const size_t* const* src_ids, size_t n_src, kvbm_layout_handle dst, const size_t* dst_ids,
                                       size_t n_dst, size_t token_begin, size_t token_end, const kvbm_head_window* windows,
                                       size_t num_windows, const kvbm_transfer_options* opts, kvbm_notification* out);

/* Layer streaming of a gather or re-paging gather: the per-layer flags, the only way to pass them to these transfers. */
typedef struct kvbm_layer_stream {
  const uint32_t* const* src_layer_ready_flags; /* [num_srcs], indexed like srcs: source s's [num_layers] ready flags; layer l of
                                                   source s is read once flag l has reached opts->epoch (kvbm_paged_copy_opts.epoch's
                                                   cyclic order) */
  size_t num_srcs;
  uint32_t* layer_done_flags;                   /* nullable, [num_layers], on the destination: entry l = epoch once layer l landed */
} kvbm_layer_stream;

/* kvbm_manager_execute_gather, streamed layer by layer: every window's layer l is read only after its source's ready flag l has
 * reached opts->epoch, and layer_done_flags[l] is written once every window's layer l landed.  A one-window plan streams a plain
 * format change (a window over every head of both sides) or a single re-shard window.  Validation is execute_gather's, with its
 * codes and texts (the options' own layer_ready_flags / layer_done_flags / per_dst_* / multicast stay rejected); before it,
 * KVBM_ERR for a NULL ls, a NULL flag table or a NULL entry, and KVBM_ERR_LENGTH_MISMATCH for ls->num_srcs != num_srcs; after
 * it, KVBM_ERR for a flag array the manager's device cannot reach: allowed are its own memory, memory of a device whose peer
 * access was enabled through kvbm_manager_enable_peer_access or by an IPC mapping this manager opened, and mapped pinned host
 * memory.  Honoured on top of execute_gather's options: epoch, gate_mode,
 * gate_timeout_ms, max_ctas and done_flag (see kvbm_permute_stream for the two gate forms).  The notification completes as a
 * gated execute_transfer's, with KVBM_ERR_TIMEOUT after the spinning form gave up on a flag.  The destination bytes and
 * bytes_moved equal execute_gather's.  At most KVBM_GATHER_MAX_HEADS covered heads, also with one window. */
int kvbm_manager_execute_gather_streamed(kvbm_transfer_manager* m, size_t num_srcs, const kvbm_layout_handle* srcs,
                                         const size_t* const* src_ids, kvbm_layout_handle dst, const size_t* dst_ids, size_t n,
                                         const kvbm_head_window* windows, size_t num_windows, const kvbm_layer_stream* ls,
                                         const kvbm_transfer_options* opts, kvbm_notification* out);

/* A PP x TP re-shard's assembly as ONE hand-off: kvbm_manager_execute_gather with a layer window per window (a
 * kvbm_tp_pp_reshard_plan passes as it is; windows[j].src_rank indexes srcs / src_ids).  Heads [src_head_begin, +head_count) of
 * layers [src_layer_begin, +layer_count) of block src_ids[src_rank][i] land as heads [dst_head_begin, +head_count) of layers
 * [dst_layer_begin, +layer_count) of block dst_ids[i]; every other destination byte keeps its value.  Windows with equal
 * destination layer windows form a stage.  The options' layer range counts destination layers, and so do cast_scales
 * ([dst num_layers * outer_dim]).  ls (nullable): streamed as kvbm_manager_execute_gather_streamed, ls->src_layer_ready_flags[s]
 * being source s's array over its own layers and layer_done_flags the destination's.  Errors, first one wins: with ls, its shape
 * as kvbm_manager_execute_gather_streamed; execute_gather's window checks, except that only windows of one stage may not
 * share a destination head, plus KVBM_ERR_RANGE a window without layers and KVBM_ERR_OVERLAP two layer windows that partly
 * overlap in the destination; KVBM_ERR_HANDLE an unknown handle; KVBM_ERR_RANGE a layer window past its source's or the
 * destination's num_layers, or a destination layer of the range that no window covers; each (source, destination) pair's checks
 * of execute_gather with the same codes and texts, except the equal layer counts; an empty block or layer range then returns
 * KVBM_OK with nothing launched; with ls,
 * its flags' reachability.  One upload, one kvbm_kernels_paged_stage_gather launch, one notification; bytes_moved counts each
 * window's destination bytes over its layers inside the range. */
int kvbm_manager_execute_stage_gather(kvbm_transfer_manager* m, size_t num_srcs, const kvbm_layout_handle* srcs,
                                      const size_t* const* src_ids, kvbm_layout_handle dst, const size_t* dst_ids, size_t n,
                                      const kvbm_shard_window* windows, size_t num_windows, const kvbm_layer_stream* ls,
                                      const kvbm_transfer_options* opts, kvbm_notification* out);

/* kvbm_manager_execute_repage_gather, streamed as kvbm_manager_execute_gather_streamed is; one window over every head of both
 * sides streams a plain re-page.  Validation is execute_repage_gather's, with the same additions. */
int kvbm_manager_execute_repage_gather_streamed(kvbm_transfer_manager* m, size_t num_srcs, const kvbm_layout_handle* srcs,
                                                const size_t* const* src_ids, size_t n_src, kvbm_layout_handle dst, const size_t* dst_ids,
                                                size_t n_dst, size_t token_begin, size_t token_end, const kvbm_head_window* windows,
                                                size_t num_windows, const kvbm_layer_stream* ls, const kvbm_transfer_options* opts,
                                                kvbm_notification* out);

/* A PP x TP re-shard's assembly across engines with different page sizes as ONE hand-off: kvbm_manager_execute_stage_gather's
 * layer windows over kvbm_manager_execute_repage_gather's token range (a kvbm_tp_pp_reshard_plan passes as it is).  Heads
 * [src_head_begin, +head_count) of layers [src_layer_begin, +layer_count) of source src_rank land as heads [dst_head_begin,
 * +head_count) of layers [dst_layer_begin, +layer_count) of the destination, at every token of [token_begin, token_end), with the
 * ids of kvbm_manager_execute_repage_gather (src_ids[s]: source s's table for Ps, n_src ids each; dst_ids: the destination's for
 * Pd).  Every other destination byte keeps its value.  All sources share one page size; each may have its own num_layers.  The
 * options' layer range counts destination layers, and so do cast_scales ([dst num_layers * outer_dim]).  ls (nullable): streamed
 * as kvbm_manager_execute_stage_gather.  Errors, first one wins: with ls, its shape as kvbm_manager_execute_gather_streamed;
 * kvbm_manager_execute_stage_gather's window checks; its KVBM_ERR_HANDLE and layer-window checks; each window's pair checks of
 * kvbm_manager_execute_repage_gather except the equal layer counts, then its one page size; its token range; the layer range
 * and cast scales against the destination; then the id counts, block ids, strategy, device, cast scales and, with ls, flag
 * reachability as kvbm_manager_execute_repage_gather (an empty token or layer range returns KVBM_OK with nothing launched).  One
 * upload, one kvbm_kernels_paged_stage_repage_gather launch (its streamed form with ls), one notification; bytes_moved counts
 * each window's destination bytes over its layers inside the range. */
int kvbm_manager_execute_stage_repage_gather(kvbm_transfer_manager* m, size_t num_srcs, const kvbm_layout_handle* srcs,
                                             const size_t* const* src_ids, size_t n_src, kvbm_layout_handle dst, const size_t* dst_ids,
                                             size_t n_dst, size_t token_begin, size_t token_end, const kvbm_shard_window* windows,
                                             size_t num_windows, const kvbm_layer_stream* ls, const kvbm_transfer_options* opts,
                                             kvbm_notification* out);

/* One sequence of kvbm_manager_execute_repage_batch: the arguments kvbm_manager_execute_stage_repage_gather takes per request. */
typedef struct kvbm_repage_batch_seq {
  size_t token_begin, token_end;
  const size_t* const* src_ids; /* [num_srcs] lists of n_src ids: source s's table[token_begin / Ps .. ceil(token_end / Ps)) */
  size_t n_src;
  const size_t* dst_ids;        /* the destination's table[token_begin / Pd .. ceil(token_end / Pd)) */
  size_t n_dst;
} kvbm_repage_batch_seq;

/* A batch of sequences as ONE hand-off (what a continuous-batching decode step admits, or a prefill batch finishes, at once):
 * kvbm_manager_execute_stage_repage_gather for every sequence of seqs[], each with its own token range and block tables, under
 * one plan, one set of options and, with ls, one set of layer flags -- one staged copy of every table and the batch's unit
 * table, one kvbm_kernels_paged_stage_repage_gather_batch launch (its streamed form with ls), one notification, and
 * options.done_flag written once, after every sequence's bytes landed.  A plan without layer windows (PP1) is windows whose
 * layer window is the identity over every layer.  With ls, layer_done_flags[l] is written once layer l of every sequence
 * landed.  Two sequences may share source blocks (a shared prefix); a destination block may appear once in the whole batch.
 * Errors: with ls, its shape; then, sequence by sequence in batch order, every check of
 * kvbm_manager_execute_stage_repage_gather with its code and text, so the first rejected sequence returns what the single call
 * would have returned for it (a batch without sequences still has its windows checked); then the concatenated destination ids
 * unique (KVBM_ERR_DUPLICATE_DST) and, where a source is the destination's layout, disjoint from its concatenated source ids
 * (KVBM_ERR_OVERLAP).  A batch whose sequences or layer range are all empty returns KVBM_OK with nothing launched.  bytes_moved
 * counts the sum of what the single calls would.  Per-sequence completion words are not provided. */
int kvbm_manager_execute_repage_batch(kvbm_transfer_manager* m, size_t num_srcs, const kvbm_layout_handle* srcs, kvbm_layout_handle dst,
                                      const kvbm_repage_batch_seq* seqs, size_t num_seqs, const kvbm_shard_window* windows,
                                      size_t num_windows, const kvbm_layer_stream* ls, const kvbm_transfer_options* opts,
                                      kvbm_notification* out);

/* kvbm_manager_execute_repage_batch between engines whose page sizes need not divide each other (a hybrid model's 544-token
 * attention block against a 64-token decode page, or 24 against 16), through kvbm_kernels_paged_stage_repage_gather_anypage, or
 * its streamed form with ls.  The arguments, plans, errors, codes, texts and their order are kvbm_manager_execute_repage_batch's,
 * but for each pair's page rule: "one page size divides the other" is not asked, and pages past the exactness bound of
 * include/kvbm_kernels.h, (big + small - gcd) * small < 2^32, fail with KVBM_ERR_UNSUPPORTED in its place.  One staged copy
 * of every table and the unit table of kvbm_kernels_repage_anypage_units, one launch, one notification, options.done_flag
 * written once; bytes_moved as the batch's.  With dividing pages the destination bytes are the batch's. */
int kvbm_manager_execute_repage_anypage(kvbm_transfer_manager* m, size_t num_srcs, const kvbm_layout_handle* srcs, kvbm_layout_handle dst,
                                        const kvbm_repage_batch_seq* seqs, size_t num_seqs, const kvbm_shard_window* windows,
                                        size_t num_windows, const kvbm_layer_stream* ls, const kvbm_transfer_options* opts,
                                        kvbm_notification* out);

/* One sequence of kvbm_manager_execute_repage_batch_routed: a kvbm_repage_batch_seq plus the sources it is read from. */
typedef struct kvbm_repage_route_seq {
  size_t token_begin, token_end;
  const size_t* const* src_ids; /* [num_srcs]; src_ids[r] (n_src ids) read only for r in src_mask, the others may be NULL */
  size_t n_src;
  const size_t* dst_ids;        /* the destination's table[token_begin / Pd .. ceil(token_end / Pd)) */
  size_t n_dst;
  uint32_t src_mask;            /* bit r: this sequence is read from srcs[r] (every window whose src_rank bit is set) */
} kvbm_repage_route_seq;

/* A decode step's new sequences, each served by its own prefill worker, as ONE hand-off: kvbm_manager_execute_repage_batch where
 * sequence i is read only through the windows whose source is in seqs[i].src_mask, through
 * kvbm_kernels_paged_stage_repage_gather_routed, or its streamed form with ls.  Under one plan that tiles one prefill group's
 * windows over several identical workers (tile_reshard_plan in Python), the windows of two workers write the same destination
 * heads; that is allowed as long as no sequence is routed to both.  Every other destination byte keeps its value.  Errors, first
 * one wins: with ls, its shape (ls->num_srcs == num_srcs, every entry non-null); the batch's window checks except that two windows
 * of one stage may share destination heads; a null sequence list; num_srcs > 32 (KVBM_ERR_UNSUPPORTED); then sequence by sequence
 * the routing: a src_mask of 0, a bit at or above num_srcs, or a bit naming a source no window reads (KVBM_ERR_RANGE), two routed
 * windows of one stage sharing a destination head (KVBM_ERR_OVERLAP), a destination layer of the range no routed window covers
 * (KVBM_ERR_RANGE); then sequence by sequence every check of kvbm_manager_execute_stage_repage_gather with its code and text, the
 * source id lists read and checked for routed sources only; last, the destination ids unique over the whole batch
 * (KVBM_ERR_DUPLICATE_DST) and, where a source is the destination's layout, disjoint from the ids of the sequences routed to it
 * (KVBM_ERR_OVERLAP).  Unrouted positions of the staged source tables hold block 0 and are never read.  bytes_moved counts the
 * routed windows' bytes only.  With ls, layer_done_flags[l] is written once layer l of every sequence landed, and only the
 * sources some sequence is routed to are waited on. */
int kvbm_manager_execute_repage_batch_routed(kvbm_transfer_manager* m, size_t num_srcs, const kvbm_layout_handle* srcs, kvbm_layout_handle dst,
                                             const kvbm_repage_route_seq* seqs, size_t num_seqs, const kvbm_shard_window* windows,
                                             size_t num_windows, const kvbm_layer_stream* ls, const kvbm_transfer_options* opts,
                                             kvbm_notification* out);

/* One prefill rank's KV to every decode rank that needs it, as ONE hand-off: the mirror image of
 * kvbm_manager_execute_stage_repage_gather.  For window w, heads [src_head_begin, +head_count) of source layers [src_layer_begin,
 * +layer_count) land as heads [dst_head_begin, +head_count) of layers [dst_layer_begin, +layer_count) of dsts[w.dst_rank], at every
 * token of [token_begin, token_end); a kvbm_tp_pp_scatter_plan passes as it is.  src_ids holds the source's table[token_begin / Ps
 * .. ceil(token_end / Ps)) (n_src ids), dst_ids[d] destination d's table[token_begin / Pd .. ceil(token_end / Pd)) (n_dst ids
 * each); every destination has the same page Pd.  Every other destination byte keeps its value.  Each source vector is read once
 * and cast once, however many windows take it (replicated heads, MLA's latent head).  The options' layer range and cast_scales
 * count SOURCE layers ([src num_layers * outer_dim]).  Honoured options: execute_repage's, plus per_dst_done_flags (indexed like
 * dsts); done_flag and the notification complete once, after every destination landed.  Errors, first one wins: KVBM_ERR no
 * destination or window, or options.head_count; KVBM_ERR_UNSUPPORTED more than KVBM_GATHER_MAX_SOURCES windows; KVBM_ERR_RANGE a
 * window naming no destination, with no heads or no layers; KVBM_ERR_OVERLAP two windows whose source layer windows partly
 * overlap, two windows of one destination whose destination (layer, head) rectangles intersect, or one handle listed twice in
 * dsts; KVBM_ERR_HANDLE an unknown handle; KVBM_ERR_RANGE a layer window past the source's or its destination's num_layers, or a
 * source layer of the range that no window covers; each (source, destination) pair's checks of
 * kvbm_manager_execute_stage_repage_gather with its codes and texts (layer streaming and multicast in the options are
 * KVBM_ERR_UNSUPPORTED there); KVBM_ERR_INCOMPATIBLE destinations with different page sizes; then the token range, the layer range
 * and cast scales against the source, the id counts, the block ids of each pair, strategy, device and cast-scale reachability as
 * there (an empty token or layer range returns KVBM_OK with nothing launched).  One staged copy of every id list, one
 * kvbm_kernels_paged_repage_scatter launch, one notification; bytes_moved counts each window's destination bytes over its layers
 * inside the range. */
int kvbm_manager_execute_repage_scatter(kvbm_transfer_manager* m, kvbm_layout_handle src, const size_t* src_ids, size_t n_src,
                                        size_t num_dsts, const kvbm_layout_handle* dsts, const size_t* const* dst_ids, size_t n_dst,
                                        size_t token_begin, size_t token_end, const kvbm_scatter_window* windows, size_t num_windows,
                                        const kvbm_transfer_options* opts, kvbm_notification* out);

/* kvbm_manager_execute_repage_scatter streamed layer by layer: a prefill rank pushes each source layer to every destination as soon
 * as its ready flag reached opts->epoch, while its forward pass computes later layers.  ls names the ONE source's flags:
 * ls->src_layer_ready_flags[0] is its [src num_layers] array, and layer_done_flags (nullable, [src num_layers]) gets entry l =
 * epoch once source layer l landed in every destination that takes it.  Errors, first one wins: KVBM_ERR for a NULL ls, a NULL
 * flag table or a NULL entry, and KVBM_ERR_LENGTH_MISMATCH for ls->num_srcs != 1; then every check of
 * kvbm_manager_execute_repage_scatter, in its order, with its codes and texts (the options' own layer flags and multicast stay
 * rejected); then KVBM_ERR for a flag array the manager's device cannot reach, as kvbm_manager_execute_gather_streamed.  Honoured
 * on top of execute_repage_scatter's options: epoch, gate_mode, gate_timeout_ms and max_ctas (see kvbm_permute_stream);
 * per_dst_done_flags and done_flag are written once, after the last byte, and not after a gate timeout.  The notification
 * completes as a gated transfer's, with KVBM_ERR_TIMEOUT after the spinning form gave up on a flag.  One staged copy of every id
 * list and the gate's workspace, one kvbm_kernels_paged_repage_scatter_streamed launch; the destination bytes and bytes_moved
 * equal execute_repage_scatter's. */
int kvbm_manager_execute_repage_scatter_streamed(kvbm_transfer_manager* m, kvbm_layout_handle src, const size_t* src_ids, size_t n_src,
                                                 size_t num_dsts, const kvbm_layout_handle* dsts, const size_t* const* dst_ids,
                                                 size_t n_dst, size_t token_begin, size_t token_end, const kvbm_scatter_window* windows,
                                                 size_t num_windows, const kvbm_layer_stream* ls, const kvbm_transfer_options* opts,
                                                 kvbm_notification* out);

/* One sequence of kvbm_manager_execute_repage_scatter_batch: the arguments kvbm_manager_execute_repage_scatter takes per request. */
typedef struct kvbm_scatter_batch_seq {
  size_t token_begin, token_end;
  const size_t* src_ids;        /* the source's table[token_begin / Ps .. ceil(token_end / Ps)) */
  size_t n_src;
  const size_t* const* dst_ids; /* [num_dsts] lists of n_dst ids: destination d's table[token_begin / Pd .. ceil(token_end / Pd)) */
  size_t n_dst;
} kvbm_scatter_batch_seq;

/* A prefill batch's sequences pushed to every decode rank that needs them, as ONE hand-off: kvbm_manager_execute_repage_scatter
 * for every sequence of seqs[], each with its own token range and block tables, under one plan (a kvbm_tp_pp_scatter_plan passes as
 * it is), one set of destinations and one set of options -- one staged copy of the source's and every destination's concatenated
 * tables, the batch's unit table and, with ls, the gate's workspace; one kvbm_kernels_paged_repage_scatter_batch launch (its
 * streamed form with ls); one notification.  ls (nullable) streams it as kvbm_manager_execute_repage_scatter_streamed does, with
 * ls->num_srcs == 1: one ready flag per source layer covers the whole batch, and layer_done_flags[l] is written once source layer l
 * of every sequence landed in every destination that takes it.  per_dst_done_flags and done_flag are written once, after every
 * sequence landed (never after a gate timeout).  Two sequences may share source blocks (a shared prefix); a destination block may
 * appear once per destination in the whole batch.  Errors, first one wins: with ls, its shape (as the streamed scatter); then,
 * sequence by sequence in batch order, every check of kvbm_manager_execute_repage_scatter (and, with ls, of its streamed form) with
 * its code and text, so the first rejected sequence returns what the single call would have returned for it (a batch without
 * sequences still has its windows checked); then, for each destination, its concatenated ids unique (KVBM_ERR_DUPLICATE_DST) and,
 * where the source is that destination's layout, disjoint from the concatenated source ids (KVBM_ERR_OVERLAP).  A batch whose
 * sequences or layer range are all empty returns KVBM_OK with nothing launched.  bytes_moved counts the sum of what the single
 * calls would.  Per-sequence completion words are not provided. */
int kvbm_manager_execute_repage_scatter_batch(kvbm_transfer_manager* m, kvbm_layout_handle src, size_t num_dsts, const kvbm_layout_handle* dsts,
                                              const kvbm_scatter_batch_seq* seqs, size_t num_seqs, const kvbm_scatter_window* windows,
                                              size_t num_windows, const kvbm_layer_stream* ls, const kvbm_transfer_options* opts,
                                              kvbm_notification* out);

/* kvbm_manager_execute_repage_scatter_batch between engines whose page sizes need not divide each other (a hybrid model's
 * 544-token attention block pushed into 64-token decode pages, or 24 into 16), through kvbm_kernels_paged_repage_scatter_anypage,
 * or its streamed form with ls.  The arguments, plans, errors, codes, texts and their order are
 * kvbm_manager_execute_repage_scatter_batch's, but for each window's page rule: "one page size divides the other" is not asked,
 * and pages past the exactness bound of include/kvbm_kernels.h, (big + small - gcd) * small < 2^32, fail with
 * KVBM_ERR_UNSUPPORTED and kvbm_manager_execute_repage_anypage's text in its place.  One staged copy of every table and the unit
 * table of kvbm_kernels_repage_anypage_units, one launch, one notification; per_dst_done_flags and done_flag written once, after
 * every sequence landed (never after a gate timeout); bytes_moved as the batch's.  With dividing pages the destination bytes are
 * the batch's.  Every other scatter entry keeps rejecting pages that do not divide. */
int kvbm_manager_execute_repage_scatter_anypage(kvbm_transfer_manager* m, kvbm_layout_handle src, size_t num_dsts,
                                                const kvbm_layout_handle* dsts, const kvbm_scatter_batch_seq* seqs, size_t num_seqs,
                                                const kvbm_scatter_window* windows, size_t num_windows, const kvbm_layer_stream* ls,
                                                const kvbm_transfer_options* opts, kvbm_notification* out);

/* One sequence of kvbm_manager_execute_repage_scatter_routed: a kvbm_scatter_batch_seq plus the destinations it goes to. */
typedef struct kvbm_scatter_route_seq {
  size_t token_begin, token_end;
  const size_t* src_ids;        /* the source's table[token_begin / Ps .. ceil(token_end / Ps)) */
  size_t n_src;
  const size_t* const* dst_ids; /* [num_dsts]; dst_ids[d] (n_dst ids) read only for d in dst_mask, the others may be NULL */
  size_t n_dst;
  uint32_t dst_mask;            /* bit d: this sequence goes to dsts[d] */
} kvbm_scatter_route_seq;

/* A prefill batch whose sequences belong to different decode workers, as ONE hand-off: kvbm_manager_execute_repage_scatter_batch
 * where sequence i lands only in the destinations of seqs[i].dst_mask (every window whose dst_rank bit is set), through
 * kvbm_kernels_paged_repage_scatter_routed, or its streamed form with ls.  Under one plan that tiles one decode group's windows over
 * several identical workers, each sequence reaches its own worker's ranks and no others.  Every other destination byte keeps its
 * value.  Errors, first one wins: with ls, its shape; the batch's window checks and a null sequence list; num_dsts > 32
 * (KVBM_ERR_UNSUPPORTED); then sequence by sequence the routing: a dst_mask of 0, a bit at or above num_dsts, or a bit naming a
 * destination no window writes (KVBM_ERR_RANGE); then sequence by sequence every check of kvbm_manager_execute_repage_scatter
 * with its code and text, the per-destination id lists read and checked for routed destinations only; last, for each destination,
 * the ids of the sequences routed to it unique (KVBM_ERR_DUPLICATE_DST) and, where the source is that destination's layout,
 * disjoint from every source id (KVBM_ERR_OVERLAP).  A destination block may thus appear in two sequences routed to different
 * destinations.  bytes_moved counts the routed windows' bytes only.  per_dst_done_flags and done_flag are written once, after the
 * last byte, never after a gate timeout. */
int kvbm_manager_execute_repage_scatter_routed(kvbm_transfer_manager* m, kvbm_layout_handle src, size_t num_dsts, const kvbm_layout_handle* dsts,
                                               const kvbm_scatter_route_seq* seqs, size_t num_seqs, const kvbm_scatter_window* windows,
                                               size_t num_windows, const kvbm_layer_stream* ls, const kvbm_transfer_options* opts,
                                               kvbm_notification* out);

/* kvbm_manager_execute_repage_scatter_routed between engines whose page sizes need not divide each other (a hybrid prefill pool's
 * 544-token blocks pushed to several decode workers with 64-token pages), through kvbm_kernels_paged_repage_scatter_routed_anypage,
 * or its streamed form with ls.  The arguments, plans, routing, errors, codes, texts and their order are
 * kvbm_manager_execute_repage_scatter_routed's, but for each window's page rule: "one page size divides the other" is not asked,
 * and pages past the exactness bound, (big + small - gcd) * small < 2^32, fail with KVBM_ERR_UNSUPPORTED and
 * kvbm_manager_execute_repage_anypage's text.  The staged unit table is kvbm_kernels_repage_route_anypage_units' over each
 * non-empty sequence's range and window mask.  With dividing pages the destination bytes are the routed scatter's. */
int kvbm_manager_execute_repage_scatter_routed_anypage(kvbm_transfer_manager* m, kvbm_layout_handle src, size_t num_dsts,
                                                       const kvbm_layout_handle* dsts, const kvbm_scatter_route_seq* seqs, size_t num_seqs,
                                                       const kvbm_scatter_window* windows, size_t num_windows, const kvbm_layer_stream* ls,
                                                       const kvbm_transfer_options* opts, kvbm_notification* out);

/* kvbm_manager_execute_repage_batch_routed between engines whose page sizes need not divide each other, through
 * kvbm_kernels_paged_stage_repage_gather_routed_anypage, or its streamed form with ls.  The arguments, plans, routing, errors,
 * codes, texts and their order are kvbm_manager_execute_repage_batch_routed's, but for each window's page rule, which is
 * kvbm_manager_execute_repage_anypage's: pages past the exactness bound fail with KVBM_ERR_UNSUPPORTED and its text.  With dividing
 * pages the destination bytes are the routed gather's. */
int kvbm_manager_execute_repage_batch_routed_anypage(kvbm_transfer_manager* m, size_t num_srcs, const kvbm_layout_handle* srcs,
                                                     kvbm_layout_handle dst, const kvbm_repage_route_seq* seqs, size_t num_seqs,
                                                     const kvbm_shard_window* windows, size_t num_windows, const kvbm_layer_stream* ls,
                                                     const kvbm_transfer_options* opts, kvbm_notification* out);

/* Completion: the transfer's last warp writes a flag in pinned host memory (no cudaEventQuery polling). */
int kvbm_notification_is_complete(kvbm_transfer_manager* m, kvbm_notification n);  /* 1 / 0 / <0 error */
int kvbm_notification_wait(kvbm_transfer_manager* m, kvbm_notification n, int64_t timeout_us);

/* ---- NVLS multicast groups: identical KV blocks to N GPUs with ONE write per tile --------------------------------
 * Replaces CollectiveOps::broadcast / the grouped ncclBcast per region (lib/kvbm-engine/src/collectives/mod.rs:75-106,
 * nccl.rs:421-462).  Every receiver binds a pool allocation of the same size to one CUmulticastObject; the sender maps
 * the object and passes a layout over that mapping with kvbm_transfer_options.multicast (host API) or
 * kvbm_paged_copy_opts.multicast (kernel ABI).  Block b of the layout lands at the same offset in every bound pool.
 * Order of calls (all participating processes): create | import_fd  ->  add_device (every device, by its owner)
 * -> [barrier] -> bind_local (each receiver) -> [barrier] -> map (the sender).  bind_local / map block inside the
 * driver until every device has been added.  Needs NVSwitch + CU_DEVICE_ATTRIBUTE_MULTICAST_SUPPORTED. */
typedef struct kvbm_mc_group kvbm_mc_group;
int kvbm_mc_supported(int device);   /* 1 / 0 (kvbm_last_error says why) */
/* bytes_per_device is rounded up to the multicast granularity (kvbm_mc_group_size).  shareable != 0 allows export_fd. */
int kvbm_mc_group_create(int num_devices, size_t bytes_per_device, int shareable, kvbm_mc_group** out);
int kvbm_mc_group_export_fd(kvbm_mc_group* g, int* fd);   /* POSIX fd; pass it to the peers over SCM_RIGHTS */
int kvbm_mc_group_import_fd(int fd, int num_devices, size_t bytes_per_device, kvbm_mc_group** out);
size_t kvbm_mc_group_size(const kvbm_mc_group* g);
int kvbm_mc_group_add_device(kvbm_mc_group* g, int device);
/* allocate this device's pool (cuMemCreate), map it for the device and bind it at offset 0 of the object */
int kvbm_mc_group_bind_local(kvbm_mc_group* g, int device, void** unicast_ptr);
/* bind the first kvbm_mc_group_size() bytes of memory the ENGINE owns (cuMulticastBindAddr): the range must be backed by the
 * driver's VMM API (cuMemCreate / cuMemMap, e.g. PyTorch expandable segments) and aligned to the multicast granularity */
int kvbm_mc_group_bind_addr(kvbm_mc_group* g, int device, void* ptr, size_t bytes);
/* map the multicast object for `device` (the sender); stores to the returned range reach every bound pool */
int kvbm_mc_group_map(kvbm_mc_group* g, int device, void** multicast_ptr);
void kvbm_mc_group_destroy(kvbm_mc_group* g);

/* accounting for the bench */
uint64_t kvbm_manager_bytes_moved(kvbm_transfer_manager* m);
uint64_t kvbm_manager_h2d_bytes(kvbm_transfer_manager* m);   /* block-table uploads */

#ifdef __cplusplus
}
#endif
#endif /* KVBM_PHYSICAL_H */
