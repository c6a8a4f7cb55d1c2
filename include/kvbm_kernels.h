/*
 * kvbm_kernels.h -- C ABI of libkvbm_kernels.so, the H100-native (sm_90a) replacement for
 * Dynamo's lib/kvbm-kernels.
 *
 * Part 1 are the six symbols the reference exports and its Rust FFI binds
 *   (/root/reference/lib/kvbm-kernels/cuda/tensor_kernels.cu:306,332,360,389,477,551;
 *    Rust declarations lib/kvbm-kernels/src/tensor_kernels.rs:46-74,89-109).
 * Signatures, enum values, return codes and edge-case behaviour are identical, so this library is a
 * drop-in via LD_LIBRARY_PATH exactly as lib/kvbm-kernels/cuda/stubs.c:4-7 documents.
 *
 * Part 2 are the v2 extensions: the block-table ("paged") gather -> push -> scatter kernel with
 * address arithmetic on the device, multi-destination fan-out over NVLink peer mappings, the fused
 * fp8<->bf16 cast and in-kernel completion / layer-streaming flags.  They replace the host loop +
 * pointer-table upload + host sync of lib/kvbm-physical/src/transfer/executor/cuda.rs:234-327 and
 * the grouped ncclBcast of lib/kvbm-engine/src/collectives/nccl.rs:321-356.
 *
 * No torch types; plain pointers and sizes.  All functions are thread-safe and hold no global state
 * (device attribute queries are cached per device).  Nothing here ever falls back to a CPU copy.
 */
#ifndef KVBM_KERNELS_H
#define KVBM_KERNELS_H

#include <stdbool.h>
#include <stddef.h>
#include <stdint.h>

#if defined(__CUDA_RUNTIME_API_H__) || defined(__DRIVER_TYPES_H__)
/* cudaError_t / cudaStream_t come from the CUDA headers */
#else
typedef int cudaError_t;    /* cudaSuccess == 0, as lib/kvbm-kernels/cuda/stubs.c:14-18 */
typedef void* cudaStream_t; /* opaque */
#endif

#ifdef __cplusplus
extern "C" {
#endif

/* ============================ Part 1: reference ABI (exact) ============================ */

/* tensor_kernels.cu:59-69 */
enum { KVBM_DTYPE_F16 = 0, KVBM_DTYPE_BF16 = 1, KVBM_DTYPE_F32 = 2, KVBM_DTYPE_F64 = 3 };
enum { KVBM_BLOCK_LAYOUT_NHD = 0, KVBM_BLOCK_LAYOUT_HND = 1 };
/* tensor_kernels.cu:371-375 */
enum {
  KVBM_MEMCPY_BATCHED_WITH_FALLBACK = 0,
  KVBM_MEMCPY_FALLBACK_ONLY = 1,
  KVBM_MEMCPY_BATCH_WITHOUT_FALLBACK = 2,
};

/* Replaces tensor_kernels.cu:551-571 (K1).  src_ptrs/dst_ptrs are DEVICE-ACCESSIBLE tables (device
 * or pinned host) of num_pairs pointers; every pair copies copy_size_bytes; any alignment; src/dst
 * may be device, peer-device or pinned-host memory.  num_pairs==0 || copy_size_bytes==0 ->
 * cudaSuccess before the NULL checks; NULL table -> cudaErrorInvalidValue. */
cudaError_t kvbm_kernels_launch_vectorized_copy(void** src_ptrs, void** dst_ptrs,
                                                size_t copy_size_bytes, int num_pairs,
                                                cudaStream_t stream);

/* Replaces tensor_kernels.cu:389-473 (K4).  HOST pointer tables, consumed before return. */
cudaError_t kvbm_kernels_memcpy_batch(const void* const* src_ptrs, void* const* dst_ptrs,
                                      size_t size_per_copy, size_t num_copies, int mode,
                                      cudaStream_t stream);

/* Replaces tensor_kernels.cu:306-330 (K2): block stacks [nl*no chunks of NHD|HND] -> universal
 * [nh,nl,no,nt,hd].  Tables are device-accessible. Unknown dtype -> cudaErrorInvalidValue. */
cudaError_t kvbm_kernels_launch_universal_from_block(void* const* universal_ptrs,
                                                     const void* const* block_ptrs,
                                                     size_t num_blocks, size_t nh, size_t nl,
                                                     size_t no, size_t nt, size_t hd, int dtype,
                                                     int layout, cudaStream_t stream);

/* Replaces tensor_kernels.cu:332-356 (K3): the inverse. */
cudaError_t kvbm_kernels_launch_block_from_universal(const void* const* universal_ptrs,
                                                     void* const* block_ptrs, size_t num_blocks,
                                                     size_t nh, size_t nl, size_t no, size_t nt,
                                                     size_t hd, int dtype, int layout,
                                                     cudaStream_t stream);

/* tensor_kernels.cu:360-368 */
bool kvbm_kernels_has_memcpy_batch_async(void);
/* tensor_kernels.cu:477-481: always false -- this is a real CUDA build. */
bool kvbm_kernels_is_stub_build(void);

/* ============================ Part 2: v2 extensions ============================ */

#define KVBM_MAX_DESTINATIONS 8
/* u32 words of kvbm_paged_copy_opts.sync_workspace for a source pool of `num_layers` layers */
#define KVBM_SYNC_WORKSPACE_WORDS(num_layers) ((num_layers) + 4)

/* Geometry of one KV pool as the kernel sees it.  It is the device form of
 * Layout::memory_region (lib/kvbm-physical/src/layout/mod.rs:73-78):
 *   addr(block, layer, outer) = layer_base[layer] + block*block_stride + outer*outer_stride
 * FullyContiguous pools (fully_contiguous.rs:158-162) set layer_base[l] = base + l*layer_stride;
 * LayerSeparate pools (layer_separate.rs:171-184) pass their per-layer allocations directly.
 * layer_base is a DEVICE-ACCESSIBLE array of num_layers addresses (uploaded once per pool). */
typedef struct kvbm_paged_layout {
  const uint64_t* layer_base;
  uint64_t block_stride;
  uint64_t outer_stride;
  uint32_t region_bytes; /* page_size * inner_dim * dtype_width_bytes */
  uint32_t num_layers;
  uint32_t outer_dim;
  uint32_t num_blocks;
} kvbm_paged_layout;

/* One destination of a transfer: its pool, the block table pair and optional in-band signals.
 * block id arrays are DEVICE-ACCESSIBLE int32[num_blocks]. */
typedef struct kvbm_paged_dst {
  kvbm_paged_layout layout;      /* layer_base may hold PEER addresses (NVLink-mapped) */
  const int32_t* src_block_ids;  /* blocks to gather from the source pool */
  const int32_t* dst_block_ids;  /* where they are scattered in this destination */
  uint32_t* done_flag;           /* nullable; set to `epoch` (st.release.sys) once every byte landed */
  uint32_t* layer_done_flags;    /* nullable; [num_layers]; entry l set to `epoch` when layer l landed */
} kvbm_paged_dst;

enum { KVBM_GATE_AUTO = 0, KVBM_GATE_SPIN = 1, KVBM_GATE_STREAM_WAIT = 2 };

enum {
  KVBM_CAST_NONE = 0,
  KVBM_CAST_FP8E4M3_TO_BF16 = 1, /* exact; NaN codes -> 0x7fc0 */
  KVBM_CAST_BF16_TO_FP8E4M3 = 2, /* round-to-nearest-even, saturate-to-finite */
};

typedef struct kvbm_paged_copy_opts {
  uint32_t epoch;                 /* value written to done flags; a ready flag has reached it iff (int32_t)(flag - epoch) >= 0,
                                     the cyclic order of CU_STREAM_WAIT_VALUE_GEQ, in both gate modes.  Epochs may wrap past
                                     0xFFFFFFFF; a flag must never lag its epoch by 2^31 or more (zeroed flags and epochs counting
                                     up from 1 satisfy that).  kvbm_kernels_wait_flag uses the same order. */
  const uint32_t* layer_ready_flags; /* nullable; [num_layers]; layer l is read only after flag l has reached epoch */
  uint32_t* sync_workspace;       /* device u32[KVBM_SYNC_WORKSPACE_WORDS(num_layers)], zeroed (left zeroed by every launch):
                                     per-layer landed-item counters, then the launch's control words (rings finished, abort,
                                     tile-scheduler tickets).  Required iff any flag or gating is used; without it the
                                     library lends the launch a slot of a small per-device pool for the tile scheduler. */
  int max_ctas;                   /* 0 = default (one CTA per SM: an SM moves at most ~50 GB/s per direction, the HBM-bound copy wants
                                     them all); smaller values leave SMs to the engine -- 16 CTAs saturate an NVLink peer */
  int warps_per_cta;              /* 0 = default (4).  Two warps -- a producer and a consumer -- form one ring. */
  int stages;                     /* 0 = default */
  int tile_bytes;                 /* 0 = default */
  int force_simt;                 /* 1 = never use the TMA path (diagnostics) */
  uint32_t* completion_flag;      /* nullable; device-visible (e.g. mapped pinned host) word set to
                                     completion_value once EVERY destination has landed: lets the host
                                     observe completion without cudaEventQuery polling */
  uint32_t completion_value;
  int stores_in_flight;           /* 0 = default (stages/2): slots that may still be draining to the destination;
                                     stages - stores_in_flight loads are kept in flight ahead */
  int cache_hint;                 /* bit0: L2 evict_first on source reads, bit1: on destination writes */
  int variant;                    /* 0 = TMA load + TMA store (default); 1 = TMA load + SIMT store from smem;
                                     2 / 3 = loads-only / stores-only DIAGNOSTICS (do not copy correctly) */
  int gate_timeout_ms;            /* gated transfers: a layer_ready wait longer than this aborts the launch (completion word
                                     becomes 0xFFFFFFFF, done flags are not written) instead of hanging the GPU; 0 = 10 s */
  int multicast;                  /* NVLS: non-zero = dsts[0].layout.layer_base[] hold NVLink MULTICAST addresses (a mapping of a
                                     CUmulticastObject, see kvbm_mc_group_* in kvbm_physical.h).  The payload is written ONCE
                                     (1 = multimem.st from shared memory, 2 = TMA bulk store) and the NVSwitch delivers it to every
                                     device bound to the object; dsts[1..] contribute only their done / layer_done flags.  This is
                                     the replacement of the grouped ncclBcast (kvbm-engine collectives/nccl.rs:421-462): egress of
                                     the source GPU is 1x the payload instead of Nx.  Requires cast_mode NONE, 16-byte strides. */
  int gate_mode;                  /* how layer_ready_flags are waited for: KVBM_GATE_AUTO (0) = warps of the ONE launch spin on
                                     the flags when the process loads CUDA modules eagerly (CUDA_MODULE_LOADING=EAGER), else
                                     the wait moves to the stream (cuStreamWaitValue32 + a single-layer launch per layer) so
                                     that nothing resident spins while some other kernel of the process is still being loaded
                                     lazily -- see kvbm_kernels_gate_would_spin(); KVBM_GATE_SPIN (1) / KVBM_GATE_STREAM_WAIT
                                     (2) force either behaviour.  gate_timeout_ms applies to the spinning form only. */
  int static_schedule;            /* diagnostics: 1 = split the tiles round-robin over the rings instead of the dynamic
                                     (ticket) tile scheduler */
  const float* cast_scales;       /* nullable; device-accessible float[num_layers * outer_dim] (the source pool's): entry
                                     l * outer_dim + o is the dequantisation scale of the FP8 side for layer l (absolute, whatever
                                     the layer range) and outer index o -- an engine's fp8 KV cache stores x / s and reads fp8 * s.
                                     fp8 -> bf16 writes bf16_rne(fp32_rn(fp8 * s)) (NaN codes -> 0x7fc0); bf16 -> fp8 writes
                                     e4m3_satfinite_rne(fp32_rn(bf16 / s)) (NaN -> 0x7f | sign), every code equal to the one IEEE
                                     division gives for 2^-60 <= |s| <= 2^60; zero, negative, non-finite or more extreme scales give
                                     unspecified codes.  s = 1 gives the unscaled bits.  Needs a cast_mode (cudaErrorInvalidValue with KVBM_CAST_NONE),
                                     num_layers <= 65536 and outer_dim <= 32768; runs the general (non-FAST) rings. */
} kvbm_paged_copy_opts;

/* Gather `num_blocks` non-contiguous blocks x layers [layer_begin, layer_end) x outer from `src`,
 * push them to `num_dsts` destinations and scatter them into their block tables, optionally casting.
 * One launch, one-sided (no receiver kernel), stream-ordered, never blocks the host.
 * When all destinations share one src_block_ids pointer the payload is read from HBM once and stored
 * num_dsts times (replicate); otherwise each destination's blocks are gathered separately. */
cudaError_t kvbm_kernels_paged_copy_v2(const kvbm_paged_layout* src, const kvbm_paged_dst* dsts,
                                       int num_dsts, int num_blocks, int layer_begin,
                                       int layer_end, int cast_mode,
                                       const kvbm_paged_copy_opts* opts, cudaStream_t stream);

/* ---- layout-transforming hand-off (TP / PP re-shard while the blocks move) ------------------------------------------------
 * KvBlockLayout (lib/kvbm-physical/src/layout/kv_block_layout.rs:40-95): the order of the four permutable dimensions of one
 * block, head_dim (one "row" of row_bytes) always innermost.  The reference selects a transform kernel for a pair of these
 * (transfer/executor/mod.rs:46-100) but never runs one inside a transfer -- validate_layout_compatibility rejects the pair
 * (executor/cuda.rs:69) and K2 / K3 are only reachable through host-built pointer tables.  Here the transform is part of the
 * paged gather -> scatter: no pointer tables, block ids resolved on the device, either pool may be a peer's (NVLink). */
enum {
  KVBM_KV_UNKNOWN = 0,
  KVBM_KV_UNIVERSAL_TP = 1,    /* [nh, nl, no, nt, hd] */
  KVBM_KV_UNIVERSAL_PP = 2,    /* [nl, nh, no, nt, hd] */
  KVBM_KV_OPERATIONAL_HND = 3, /* [nl, no, nh, nt, hd] */
  KVBM_KV_OPERATIONAL_NHD = 4, /* [nl, no, nt, nh, hd] */
  KVBM_KV_CUSTOM = 5,          /* named by the wire format only; no kernel */
};

typedef struct kvbm_permute_side {
  kvbm_paged_layout layout;  /* operational formats: any paged pool, the (block, layer, outer) region holds [nt, nh, hd] or
                                [nh, nt, hd].  Universal formats: the pool must be fully contiguous -- layer_base[0] +
                                id * block_stride is the start of num_layers * outer_dim * region_bytes contiguous bytes */
  const int32_t* block_ids;  /* device-accessible int32[num_blocks] */
  int kv_layout;             /* KVBM_KV_* (1..4) */
} kvbm_permute_side;

/* Block src.block_ids[i] of `src` -> block dst.block_ids[i] of `dst`, layers [layer_begin, layer_end), every element moved
 * from its position under src.kv_layout to its position under dst.kv_layout (equal layouts = plain copy).  Both sides must
 * agree on num_layers, outer_dim and region_bytes = page_size * num_heads * row_bytes; row_bytes (head_dim * element size)
 * must be a multiple of 16 in 16..65536 (powers of two take the shift-and-mask walk) and every stride a multiple of 16
 * (cudaErrorInvalidValue otherwise).  `done_flag`
 * (nullable, device-visible) receives `epoch` with system scope after the last byte landed, `completion_flag` likewise
 * `completion_value` (a one-thread signal launch behind the permuting launch; none when both are NULL).  Stream-ordered. */
cudaError_t kvbm_kernels_paged_permute(const kvbm_permute_side* src, const kvbm_permute_side* dst, int num_blocks,
                                       int layer_begin, int layer_end, uint32_t num_heads, uint32_t page_size,
                                       uint32_t row_bytes, uint32_t* done_flag, uint32_t epoch, uint32_t* completion_flag,
                                       uint32_t completion_value, cudaStream_t stream);

/* kvbm_kernels_paged_permute with the fp8 e4m3 <-> bf16 cast of kvbm_kernels_paged_copy_v2 fused in: the same walk, one launch,
 * bits identical to the paged copy's cast (fp8 NaN codes -> 0x7fc0; bf16 -> fp8 round-to-nearest-even, saturating to +-448,
 * NaN -> 0x7f with its sign).  src_row_bytes is the SOURCE row (head_dim * source element size); the destination row is twice
 * it for KVBM_CAST_FP8E4M3_TO_BF16, half of it for KVBM_CAST_BF16_TO_FP8E4M3 (src_row_bytes must then be even) and equal for
 * KVBM_CAST_NONE, which is exactly kvbm_kernels_paged_permute.  Each side's region_bytes must be page_size * num_heads * its
 * own row.  With a cast the fp8 side's row must be a multiple of 16 in 16..65536 (head_dim a multiple of 16); the walk moves
 * 16 e4m3 codes / 32 B of bf16 per vector.  An unknown cast_mode is cudaErrorInvalidValue; the zero-count early return (which
 * still signals), the stride, index-range and grid rules and the signals are those of kvbm_kernels_paged_permute. */
cudaError_t kvbm_kernels_paged_permute_cast(const kvbm_permute_side* src, const kvbm_permute_side* dst, int num_blocks,
                                            int layer_begin, int layer_end, uint32_t num_heads, uint32_t page_size,
                                            uint32_t src_row_bytes, int cast_mode, uint32_t* done_flag, uint32_t epoch,
                                            uint32_t* completion_flag, uint32_t completion_value, cudaStream_t stream);

/* kvbm_kernels_paged_permute_cast over a head window on each side (a tensor-parallel re-shard): head src_head_begin + j of
 * source block src->block_ids[i] lands as head dst_head_begin + j of destination block dst->block_ids[i], for j < head_count,
 * every layer of [layer_begin, layer_end), every outer index and token, re-ordered from the source format to the destination
 * format and cast as cast_mode says.  Every destination byte outside the window keeps its value.  Each side has its own head
 * count: its region_bytes must be page_size * its num_heads * its row, and its strides are those of its own head count.
 * head_count == 0 or a window past either side's num_heads is cudaErrorInvalidValue; every other rule (rows, cast, strides,
 * grid bounds, the zero-count early return that still signals) is kvbm_kernels_paged_permute_cast's, which is this call with
 * the full window (begin 0, count num_heads on both sides). */
cudaError_t kvbm_kernels_paged_permute_heads(const kvbm_permute_side* src, const kvbm_permute_side* dst, int num_blocks,
                                             int layer_begin, int layer_end, uint32_t src_num_heads, uint32_t src_head_begin,
                                             uint32_t dst_num_heads, uint32_t dst_head_begin, uint32_t head_count,
                                             uint32_t page_size, uint32_t src_row_bytes, int cast_mode, uint32_t* done_flag,
                                             uint32_t epoch, uint32_t* completion_flag, uint32_t completion_value,
                                             cudaStream_t stream);

/* kvbm_kernels_paged_permute_heads with the fp8 side's per-(layer, outer) dequantisation scales applied by the cast: cast_scales
 * (nullable) is a device-accessible float[num_layers * outer_dim] with the meaning, the formulas and the bits of
 * kvbm_paged_copy_opts.cast_scales.  NULL is exactly kvbm_kernels_paged_permute_heads.  Scales with KVBM_CAST_NONE are
 * cudaErrorInvalidValue, returned before any CUDA call. */
cudaError_t kvbm_kernels_paged_permute_heads_scaled(const kvbm_permute_side* src, const kvbm_permute_side* dst, int num_blocks,
                                                    int layer_begin, int layer_end, uint32_t src_num_heads, uint32_t src_head_begin,
                                                    uint32_t dst_num_heads, uint32_t dst_head_begin, uint32_t head_count,
                                                    uint32_t page_size, uint32_t src_row_bytes, int cast_mode, const float* cast_scales,
                                                    uint32_t* done_flag, uint32_t epoch, uint32_t* completion_flag,
                                                    uint32_t completion_value, cudaStream_t stream);

/* One source of kvbm_kernels_paged_permute_gather: a pool side with its own head count and one head window into the
 * destination.  A pool may appear in several sources (with different windows). */
typedef struct kvbm_permute_source {
  kvbm_permute_side side;  /* side.block_ids: int32[num_blocks], block i lands in the destination's block_ids[i] */
  uint32_t num_heads;      /* this source's heads per block (its region_bytes = page_size * num_heads * src_row_bytes) */
  uint32_t src_head_begin, dst_head_begin, head_count;
} kvbm_permute_source;

#define KVBM_GATHER_MAX_SOURCES 16
#define KVBM_GATHER_MAX_HEADS 256

/* A gather (a decode rank assembling its re-sharded heads from several source ranks): for every source s, head
 * src_head_begin + j of srcs[s].side.block_ids[i] lands as head dst_head_begin + j of dst->block_ids[i], for j < head_count,
 * every layer of [layer_begin, layer_end), re-ordered and cast as kvbm_kernels_paged_permute_heads would -- but as ONE
 * permuting launch over all sources, then one signal launch that writes done_flag / completion_flag once, after every
 * source's bytes landed.  Every destination byte outside the union of the windows keeps its value.  All sources share
 * page_size, src_row_bytes and cast_mode; each has its own format, pool and head count.  cudaErrorInvalidValue for:
 * num_srcs outside 1..KVBM_GATHER_MAX_SOURCES, a null srcs / dst / table, head_count == 0 or a window past either side's
 * heads, two windows overlapping in the destination, more than KVBM_GATHER_MAX_HEADS destination heads covered, a source
 * whose num_layers / outer_dim differ from the destination's, and every rule of kvbm_kernels_paged_permute_heads (rows,
 * cast, strides, grid bounds) applied to each (source, destination) pair.  The zero-count early return still signals. */
cudaError_t kvbm_kernels_paged_permute_gather(const kvbm_permute_source* srcs, int num_srcs, const kvbm_permute_side* dst,
                                              uint32_t dst_num_heads, int num_blocks, int layer_begin, int layer_end,
                                              uint32_t page_size, uint32_t src_row_bytes, int cast_mode, uint32_t* done_flag,
                                              uint32_t epoch, uint32_t* completion_flag, uint32_t completion_value,
                                              cudaStream_t stream);

/* kvbm_kernels_paged_permute_gather with scales, as kvbm_kernels_paged_permute_heads_scaled: ONE cast_scales array for every
 * source (per-tensor scales from a checkpoint are the same on every TP rank), indexed by the absolute layer and outer index. */
cudaError_t kvbm_kernels_paged_permute_gather_scaled(const kvbm_permute_source* srcs, int num_srcs, const kvbm_permute_side* dst,
                                                     uint32_t dst_num_heads, int num_blocks, int layer_begin, int layer_end,
                                                     uint32_t page_size, uint32_t src_row_bytes, int cast_mode, const float* cast_scales,
                                                     uint32_t* done_flag, uint32_t epoch, uint32_t* completion_flag,
                                                     uint32_t completion_value, cudaStream_t stream);

/* Re-paging: tokens [token_begin, token_end) of one sequence between two block tables with different page sizes (a prefill
 * engine's pages to a decode engine's), re-ordered from src->kv_layout to dst->kv_layout and cast as cast_mode says (bits
 * identical to kvbm_kernels_paged_permute_heads_scaled; cast_scales as there, indexed by the absolute layer and outer index).
 * Sequence token p sits in slot p % P of block table[p / P] on a side whose page is P, so src->block_ids holds
 * src_table[token_begin / Ps .. ceil(token_end / Ps)) and dst->block_ids dst_table[token_begin / Pd .. ceil(token_end / Pd)).
 * Every layer of [layer_begin, layer_end), outer index and head of each token in the range moves; every other destination byte
 * keeps its value, including the slots of the first and last destination blocks outside the range.  One page size must
 * divide the other (equal sizes are a token-range copy); both must be non-zero.  Each side's region_bytes must be its page *
 * num_heads * its row, both sides share num_layers and outer_dim, both formats must be named (KVBM_KV_* 1..4), the row, cast
 * and stride rules are kvbm_kernels_paged_permute_cast's, and the range's last block of the larger page must end below 2^32
 * tokens.  Anything else is cudaErrorInvalidValue, returned before any CUDA call.  An empty token or layer range moves nothing
 * and still signals; done_flag / completion_flag are written as kvbm_kernels_paged_permute_cast writes them. */
cudaError_t kvbm_kernels_paged_repage(const kvbm_permute_side* src, uint32_t src_page_size, const kvbm_permute_side* dst,
                                      uint32_t dst_page_size, uint32_t token_begin, uint32_t token_end, int layer_begin,
                                      int layer_end, uint32_t num_heads, uint32_t src_row_bytes, int cast_mode,
                                      const float* cast_scales, uint32_t* done_flag, uint32_t epoch, uint32_t* completion_flag,
                                      uint32_t completion_value, cudaStream_t stream);

/* Re-paging and the gather in one launch (a decode rank assembling its re-sharded heads from source ranks whose engine has another
 * page size): for every source s, head src_head_begin + j of srcs[s] lands as head dst_head_begin + j of the destination, for
 * j < head_count, at every token of [token_begin, token_end), every layer of [layer_begin, layer_end) and every outer index,
 * re-ordered and cast as kvbm_kernels_paged_permute_heads_scaled would, with the same bits.  Tokens sit as in
 * kvbm_kernels_paged_repage: srcs[s].side.block_ids holds that source's table[token_begin / Ps .. ceil(token_end / Ps)),
 * dst->block_ids the destination's table[token_begin / Pd .. ceil(token_end / Pd)).  All sources share src_page_size (Ps),
 * src_row_bytes and cast_mode; each has its own pool, format and num_heads (its region_bytes = Ps * num_heads * src_row_bytes);
 * the destination's region_bytes is Pd * dst_num_heads * its row.  cast_scales (nullable): one array for every source, indexed
 * by the absolute layer and outer index.  Every other destination byte keeps its value: heads outside the union of the windows,
 * and the slots of the first and last destination blocks outside the range.  cudaErrorInvalidValue, returned before any CUDA
 * call, for every rule of kvbm_kernels_paged_permute_gather's sources and windows and of kvbm_kernels_paged_repage's pages,
 * ranges, rows and strides.  One launch, then one signal launch that writes done_flag / completion_flag once; an empty token or
 * layer range launches nothing and still signals. */
cudaError_t kvbm_kernels_paged_repage_gather(const kvbm_permute_source* srcs, int num_srcs, uint32_t src_page_size,
                                             const kvbm_permute_side* dst, uint32_t dst_num_heads, uint32_t dst_page_size,
                                             uint32_t token_begin, uint32_t token_end, int layer_begin, int layer_end,
                                             uint32_t src_row_bytes, int cast_mode, const float* cast_scales, uint32_t* done_flag,
                                             uint32_t epoch, uint32_t* completion_flag, uint32_t completion_value,
                                             cudaStream_t stream);

/* ---- layer streaming of the layout-transforming hand-offs ------------------------------------------------------------------
 * The gate of kvbm_kernels_paged_permute_gather_streamed / kvbm_kernels_paged_repage_gather_streamed.  Layer l of source s
 * (srcs[] index) is read only after layer_ready_flags[s][l] has reached `epoch` (the cyclic order of kvbm_paged_copy_opts.epoch).
 * One CTA writes every window of a destination unit, so a unit at layer l waits for flag l of EVERY source.
 *
 * Two forms, chosen by gate_mode with kvbm_paged_copy_opts.gate_mode's rule (KVBM_GATE_AUTO spins only under eager module
 * loading, and falls back to spinning when stream memory operations are missing; KVBM_GATE_STREAM_WAIT without them is
 * cudaErrorNotSupported):
 *  - spinning: ONE launch of a persistent grid of max_ctas CTAs (0 = half the SMs) that claims batches of (block, layer,
 *    outer) units in layer-major order from the workspace's ticket word, waits once per layer it enters (gate_timeout_ms, 0 = 10 s: a longer
 *    wait aborts the transfer: done_flag is not written and completion_flag becomes 0xFFFFFFFF), publishes each finished unit
 *    before it waits on a later layer, and writes the done flags itself -- no trailing signal launch.  Needs sync_workspace.
 *  - stream-wait: per layer, cuStreamWaitValue32 (GEQ) on each source's flag, the unstreamed launch over [l, l + 1) and a
 *    one-thread signal launch; nothing resident spins.  max_ctas, gate_timeout_ms and sync_workspace do not apply.  The wait has
 *    no timeout, and it holds the device's hardware queue that `stream` maps to, not just `stream`: when the process uses more
 *    streams than the device has queues (CUDA_DEVICE_MAX_CONNECTIONS, 8 by default), a producer stream that shares the queue
 *    and releases the flags later never runs.  Release the flags from another process or device, from a stream created before
 *    the others share queues, or raise CUDA_DEVICE_MAX_CONNECTIONS.
 * Either way layer_done_flags[l] is written (epoch, system scope) once every byte of layer l landed, and done_flag (epoch) /
 * completion_flag (completion_value) after the last byte.  The destination bytes are those of the unstreamed entry. */
typedef struct kvbm_permute_stream {
  const uint32_t* layer_ready_flags[KVBM_GATHER_MAX_SOURCES]; /* per source (srcs[] index), [num_layers] each; non-null for s < num_srcs */
  uint32_t* layer_done_flags; /* nullable, [num_layers], the destination's: entry l = epoch once layer l landed */
  uint32_t* done_flag;        /* nullable */
  uint32_t epoch;
  uint32_t* sync_workspace;   /* device u32[KVBM_SYNC_WORKSPACE_WORDS(num_layers)], zeroed, left zeroed (spinning form) */
  uint32_t* completion_flag;  /* nullable */
  uint32_t completion_value;
  int gate_mode;              /* KVBM_GATE_AUTO / SPIN / STREAM_WAIT */
  int gate_timeout_ms;        /* spinning form only; 0 = 10 s */
  int max_ctas;               /* spinning form only: persistent grid size, 0 = half the SMs.  A spinning CTA holds its SM for the
                                 whole prefill, and an SM running one may not take another kernel's CTA (with a spinning CTA on
                                 every SM of an H100 a producer's layer kernel never started): values near the SM count can
                                 starve a producer on the same GPU until the gate times out */
} kvbm_permute_stream;

/* kvbm_kernels_paged_permute_gather_scaled, streamed layer by layer behind `st`'s ready flags.  One source with a full window is a
 * format change (with or without a cast), one source with a partial window a re-shard, several sources a gather; the destination
 * bytes equal the unstreamed call's bit for bit.  Every argument rule of kvbm_kernels_paged_permute_gather_scaled applies (its
 * KVBM_GATHER_MAX_HEADS covered heads also to one source).  cudaErrorInvalidValue, before any CUDA call, also for a null `st`, a
 * null ready-flag array of a used source, a gate_mode out of range and the spinning form without sync_workspace (KVBM_GATE_SPIN
 * before any CUDA call; KVBM_GATE_AUTO once it has chosen that form).  An empty block or layer range waits for nothing and writes
 * done_flag and completion_flag at once, as the unstreamed entry does; it writes no layer_done_flags. */
cudaError_t kvbm_kernels_paged_permute_gather_streamed(const kvbm_permute_source* srcs, int num_srcs, const kvbm_permute_side* dst,
                                                       uint32_t dst_num_heads, int num_blocks, int layer_begin, int layer_end,
                                                       uint32_t page_size, uint32_t src_row_bytes, int cast_mode, const float* cast_scales,
                                                       const kvbm_permute_stream* st, cudaStream_t stream);

/* kvbm_kernels_paged_repage_gather, streamed as kvbm_kernels_paged_permute_gather_streamed is.  One source with a full window is
 * kvbm_kernels_paged_repage.  Its argument rules are kvbm_kernels_paged_repage_gather's plus the gate's above. */
cudaError_t kvbm_kernels_paged_repage_gather_streamed(const kvbm_permute_source* srcs, int num_srcs, uint32_t src_page_size,
                                                      const kvbm_permute_side* dst, uint32_t dst_num_heads, uint32_t dst_page_size,
                                                      uint32_t token_begin, uint32_t token_end, int layer_begin, int layer_end,
                                                      uint32_t src_row_bytes, int cast_mode, const float* cast_scales,
                                                      const kvbm_permute_stream* st, cudaStream_t stream);

/* ---- the staged gather: a pipeline-parallel re-shard ------------------------------------------------------------------------
 * One source of kvbm_kernels_paged_stage_gather: a gather source (its side with the source pool's OWN layout.num_layers, head
 * count and head window) plus a layer window: source layers [src_layer_begin, src_layer_begin + layer_count) land as destination
 * layers [dst_layer_begin, dst_layer_begin + layer_count).  A prefill engine with pipeline parallelism has one pool per stage,
 * holding only that stage's layers; its layer 0 is the stage's first layer. */
typedef struct kvbm_stage_source {
  kvbm_permute_source src;
  uint32_t src_layer_begin, dst_layer_begin, layer_count;
} kvbm_stage_source;

/* kvbm_kernels_paged_permute_gather_scaled with a layer window per source (a decode rank assembling its layers and heads from a
 * PP x TP prefill group) in ONE launch, then one signal launch.  Sources whose layer windows are equal in the destination form a
 * stage; for every destination layer l of [layer_begin, layer_end) and every source s of l's stage, head src_head_begin + j of
 * srcs[s] at source layer l - dst_layer_begin + src_layer_begin lands as head dst_head_begin + j at destination layer l,
 * re-ordered and cast as kvbm_kernels_paged_permute_heads_scaled would, with the same bits.  Every other destination byte keeps
 * its value.  cast_scales (nullable): one float[dst num_layers * outer_dim] array indexed by the DESTINATION layer and outer index.
 * cudaErrorInvalidValue, before any CUDA call, for: num_srcs outside 1..KVBM_GATHER_MAX_SOURCES; layer_count == 0 or a window past
 * its source's num_layers or the destination's; two layer windows that overlap in the destination without being equal; a
 * destination layer of [layer_begin, layer_end) that no stage covers (stages may extend past the range); two head windows of one
 * stage that overlap in the destination (those of different stages may); more than KVBM_GATHER_MAX_HEADS covered heads counted
 * over all stages; and every other rule of kvbm_kernels_paged_permute_gather_scaled but the equal layer counts (outer_dim,
 * page_size, rows, cast, strides are shared by all sources).  An empty block or layer range moves nothing and still signals.
 * When every window is the identity over a source whose num_layers is the destination's, this is
 * kvbm_kernels_paged_permute_gather_scaled. */
cudaError_t kvbm_kernels_paged_stage_gather(const kvbm_stage_source* srcs, int num_srcs, const kvbm_permute_side* dst,
                                            uint32_t dst_num_heads, int num_blocks, int layer_begin, int layer_end, uint32_t page_size,
                                            uint32_t src_row_bytes, int cast_mode, const float* cast_scales, uint32_t* done_flag,
                                            uint32_t epoch, uint32_t* completion_flag, uint32_t completion_value, cudaStream_t stream);

/* kvbm_kernels_paged_stage_gather streamed as kvbm_kernels_paged_permute_gather_streamed is, with these flag conventions:
 * st->layer_ready_flags[s] is source s's array over ITS OWN layers ([srcs[s].src.side.layout.num_layers]), and a unit of
 * destination layer l waits only for the sources of l's stage, each at its own layer; layer_done_flags and sync_workspace are the
 * destination's ([dst num_layers]).  The argument rules are kvbm_kernels_paged_stage_gather's plus the gate's. */
cudaError_t kvbm_kernels_paged_stage_gather_streamed(const kvbm_stage_source* srcs, int num_srcs, const kvbm_permute_side* dst,
                                                     uint32_t dst_num_heads, int num_blocks, int layer_begin, int layer_end,
                                                     uint32_t page_size, uint32_t src_row_bytes, int cast_mode, const float* cast_scales,
                                                     const kvbm_permute_stream* st, cudaStream_t stream);

/* kvbm_kernels_paged_stage_gather with kvbm_kernels_paged_repage_gather's token range (a decode rank assembling its layers and heads
 * from a PP x TP prefill group whose engine has another page size) in ONE launch, then one signal launch.  For every destination
 * layer l of [layer_begin, layer_end) and every source s of l's stage, head src_head_begin + j of srcs[s] at source layer
 * l - dst_layer_begin + src_layer_begin lands as head dst_head_begin + j at destination layer l, at every token of
 * [token_begin, token_end) and every outer index, re-ordered and cast as kvbm_kernels_paged_repage_gather would, with the same bits.
 * Tokens sit as in kvbm_kernels_paged_repage: srcs[s].src.side.block_ids holds source s's table[token_begin / Ps ..
 * ceil(token_end / Ps)), dst->block_ids the destination's table for Pd.  All sources share src_page_size (Ps), src_row_bytes and
 * cast_mode; each has its own pool, format, num_heads and num_layers.  cast_scales (nullable): one float[dst num_layers *
 * outer_dim] array indexed by the DESTINATION layer and outer index.  Every other destination byte keeps its value: heads outside
 * the windows of a layer's stage, and the slots of the first and last destination blocks outside the range.
 * cudaErrorInvalidValue, before any CUDA call, for every rule of kvbm_kernels_paged_stage_gather's sources, stages and windows
 * and of kvbm_kernels_paged_repage's pages, ranges, rows and strides.  An empty token or layer range moves nothing and still
 * signals.  When every window is the identity over a source whose num_layers is the destination's, this is
 * kvbm_kernels_paged_repage_gather. */
cudaError_t kvbm_kernels_paged_stage_repage_gather(const kvbm_stage_source* srcs, int num_srcs, uint32_t src_page_size,
                                                   const kvbm_permute_side* dst, uint32_t dst_num_heads, uint32_t dst_page_size,
                                                   uint32_t token_begin, uint32_t token_end, int layer_begin, int layer_end,
                                                   uint32_t src_row_bytes, int cast_mode, const float* cast_scales, uint32_t* done_flag,
                                                   uint32_t epoch, uint32_t* completion_flag, uint32_t completion_value,
                                                   cudaStream_t stream);

/* kvbm_kernels_paged_stage_repage_gather streamed with kvbm_kernels_paged_stage_gather_streamed's flag conventions:
 * st->layer_ready_flags[s] runs over source s's OWN layers, a unit of destination layer l waits only for the sources of l's stage,
 * each at its own layer, and layer_done_flags and sync_workspace are the destination's.  The argument rules are
 * kvbm_kernels_paged_stage_repage_gather's plus the gate's. */
cudaError_t kvbm_kernels_paged_stage_repage_gather_streamed(const kvbm_stage_source* srcs, int num_srcs, uint32_t src_page_size,
                                                            const kvbm_permute_side* dst, uint32_t dst_num_heads, uint32_t dst_page_size,
                                                            uint32_t token_begin, uint32_t token_end, int layer_begin, int layer_end,
                                                            uint32_t src_row_bytes, int cast_mode, const float* cast_scales,
                                                            const kvbm_permute_stream* st, cudaStream_t stream);

/* ---- a batch of sequences in one re-paging launch ---------------------------------------------------------------------------
 * A decode step admits many requests, each with its own prefix-cache hit (its own token_begin, often inside a block), length
 * and block tables.  A batch moves them in ONE launch with one signal.  Sequence i is the range [token_begin, token_end) that
 * kvbm_kernels_paged_stage_repage_gather takes, and every side's block table is the concatenation, in batch order, of the tables
 * the single entry would take: sequence i contributes its table[token_begin / P .. ceil(token_end / P)) for the side's page P
 * (nothing when its range is empty).  All sources share Ps, so every source's concatenated table has the same per-sequence
 * offsets. */
typedef struct kvbm_repage_seq {
  uint32_t token_begin, token_end;
} kvbm_repage_seq;

/* One block of the larger-page side (the source's on a tie), in batch order; record j belongs to entry j of that side's
 * concatenated table.  q0: the slot of the block's first token inside the sequence's range; tokens: how many of its tokens lie in
 * the range; small_k: the entry of the smaller-page side's concatenated table that holds the block's first small block -- when
 * those first small blocks lie before the range it wraps below 0 in uint32 and small_k + b wraps back for every small block b the
 * range touches; seq: the sequence the block belongs to (not read by the kernels).  The routed scatter entries take
 * kvbm_route_unit instead: the same record with the sequence's target mask, which the kernels read, in place of seq. */
typedef struct kvbm_repage_unit {
  uint32_t q0, tokens, small_k, seq;
} kvbm_repage_unit;

/* Host-only (no GPU): the unit table of a batch and the lengths of its concatenated tables.  Writes min(*num_units, cap) records
 * to out (out may be NULL when cap is 0: a sizing call) and always the three counts: *num_units records, *src_ids / *dst_ids
 * entries in each source's / the destination's concatenated table.  Returns non-zero, writing nothing, for a null seqs with
 * num_seqs > 0, a page of 0, pages of which neither divides the other, big_page * small_page >= 2^32, a reversed range, or a
 * sequence whose last block of the larger page ends at or past 2^32 tokens. */
int kvbm_kernels_repage_batch_units(const kvbm_repage_seq* seqs, size_t num_seqs, uint32_t src_page_size, uint32_t dst_page_size,
                                    kvbm_repage_unit* out, size_t cap, size_t* num_units, size_t* src_ids, size_t* dst_ids);

/* kvbm_kernels_paged_stage_repage_gather over a batch: sources, stages, head windows, layer range, formats, cast and scales are
 * the launch's, as there; the token ranges are `seqs` (host memory) and the tables are concatenated as above.  `units` is
 * device-accessible memory holding what kvbm_kernels_repage_batch_units produced for the same seqs and pages; like the block
 * ids it is the caller's memory, read by the kernel and not on the host, and must stay valid until the launch has run.
 * cudaErrorInvalidValue, before any CUDA call, for: every rule of kvbm_kernels_paged_stage_repage_gather's sources, stages,
 * windows, pages, rows, cast and strides; a null seqs with num_seqs > 0; any rule of kvbm_kernels_repage_batch_units; a
 * num_units other than the helper's count; a null units with num_units > 0; num_units * layers * outer_dim of 2^31 or more.
 * Two sequences may share SOURCE blocks (a shared prefix).  Two sequences must not share a DESTINATION block: the entry cannot
 * read device ids, so this is the caller's rule.  A batch always runs the gather kernels, also for one full-window source.
 * One signal for the batch: done_flag / completion_flag are written once, after every sequence's bytes landed; per-sequence
 * completion words are not provided.  num_seqs == 0, only empty ranges, or an empty layer range move nothing and still
 * signal.  A batch of one sequence writes exactly the bytes of kvbm_kernels_paged_stage_repage_gather with that range, and a
 * batch of n the bytes of n such launches in any order. */
cudaError_t kvbm_kernels_paged_stage_repage_gather_batch(const kvbm_stage_source* srcs, int num_srcs, uint32_t src_page_size,
                                                         const kvbm_permute_side* dst, uint32_t dst_num_heads, uint32_t dst_page_size,
                                                         const kvbm_repage_seq* seqs, size_t num_seqs, const kvbm_repage_unit* units,
                                                         size_t num_units, int layer_begin, int layer_end, uint32_t src_row_bytes,
                                                         int cast_mode, const float* cast_scales, uint32_t* done_flag, uint32_t epoch,
                                                         uint32_t* completion_flag, uint32_t completion_value, cudaStream_t stream);

/* The batch streamed with kvbm_kernels_paged_stage_repage_gather_streamed's flag conventions.  A prefill batch computes layer l
 * for all its sequences together, so one ready flag per (source, layer) covers the batch, and layer_done_flags[l] is written once
 * layer l of EVERY sequence landed.  The argument rules are the batch's plus the gate's; a batch that moves nothing waits for
 * nothing, writes done_flag / completion_flag at once and no layer_done_flags. */
cudaError_t kvbm_kernels_paged_stage_repage_gather_batch_streamed(const kvbm_stage_source* srcs, int num_srcs, uint32_t src_page_size,
                                                                  const kvbm_permute_side* dst, uint32_t dst_num_heads,
                                                                  uint32_t dst_page_size, const kvbm_repage_seq* seqs, size_t num_seqs,
                                                                  const kvbm_repage_unit* units, size_t num_units, int layer_begin,
                                                                  int layer_end, uint32_t src_row_bytes, int cast_mode,
                                                                  const float* cast_scales, const kvbm_permute_stream* st,
                                                                  cudaStream_t stream);

/* ---- the re-paging scatter: one prefill rank's KV to every decode rank that needs it ------------------------------------------
 * The mirror image of kvbm_kernels_paged_stage_repage_gather: ONE source pool writes into up to KVBM_GATHER_MAX_SOURCES targets.
 * A target is one destination pool's side plus one head window (source heads [src_head_begin, +head_count) land as destination
 * heads [dst_head_begin, +head_count)) and one layer window (source layers [src_layer_begin, +layer_count) land as destination
 * layers [dst_layer_begin, +layer_count)); a pool may appear in several targets.  Targets with equal source layer windows form a
 * stage.  side.block_ids holds the target's table[token_begin / Pd .. ceil(token_end / Pd)); side.layout.num_layers is the pool's
 * own.  done_flag (nullable) receives epoch with system scope once the launch's bytes landed; targets of one pool may share it. */
typedef struct kvbm_scatter_target {
  kvbm_permute_side side;   /* destination pool, format, table for Pd over the range */
  uint32_t num_heads;       /* this destination's heads per block (its region_bytes = Pd * num_heads * its row) */
  uint32_t src_head_begin, dst_head_begin, head_count;
  uint32_t src_layer_begin, dst_layer_begin, layer_count;
  uint32_t* done_flag;      /* nullable */
} kvbm_scatter_target;

/* One source (src: its pool, format and table[token_begin / Ps .. ceil(token_end / Ps)), src_num_heads heads per block, page Ps)
 * into num_targets targets of one page Pd, in ONE launch, then one signal launch that writes every target's done_flag and
 * completion_flag (completion_value).  Each 16 B source vector is loaded once and cast once, then stored to every target of its
 * layer's stage that covers its head: replicated heads (dst_tp > num_kv_heads, MLA's one latent head) are read once.  The
 * destination bytes equal those of num_targets separate kvbm_kernels_paged_stage_repage_gather launches, bit for bit: launch t has
 * the source as its one stage source with target t's windows, over the destination image of source layers [layer_begin,
 * layer_end) under t's layer window, with cast_scales re-indexed to destination layers.  Every other destination byte keeps its
 * value.  The token range, the cast and src_row_bytes are shared; layer_begin / layer_end count SOURCE layers, and cast_scales
 * (nullable) is the SOURCE's float[src num_layers * outer_dim], indexed by the source layer and outer index.
 * cudaErrorInvalidValue, before any CUDA call, for: every page, range, row, stride and cast rule of
 * kvbm_kernels_paged_stage_repage_gather; num_targets outside 1..KVBM_GATHER_MAX_SOURCES; an empty head or layer window, or one
 * past the source's or its destination's heads or layers; two stages whose source layer windows overlap without being equal; a
 * source layer of [layer_begin, layer_end) that no stage covers; more than KVBM_GATHER_MAX_HEADS (target, head) pairs over all
 * stages; two targets with the same side.layout.layer_base and side.block_ids pointers whose destination (layer, head) rectangles
 * overlap.  The entry cannot read device ids, so for targets that share a pool through different tables, keeping their
 * destination blocks disjoint is the caller's rule.  An empty token or layer range moves nothing and still signals. */
cudaError_t kvbm_kernels_paged_repage_scatter(const kvbm_permute_side* src, uint32_t src_num_heads, uint32_t src_page_size,
                                              const kvbm_scatter_target* targets, int num_targets, uint32_t dst_page_size,
                                              uint32_t token_begin, uint32_t token_end, int layer_begin, int layer_end,
                                              uint32_t src_row_bytes, int cast_mode, const float* cast_scales, uint32_t epoch,
                                              uint32_t* completion_flag, uint32_t completion_value, cudaStream_t stream);

/* kvbm_kernels_paged_repage_scatter streamed layer by layer behind the source's ready flags, as
 * kvbm_kernels_paged_permute_gather_streamed is: a prefill rank pushes each layer to every target while its forward pass is still
 * computing later ones.  The bytes are the unstreamed call's, bit for bit; only the time at which each layer is read changes.
 * Flag conventions, all in SOURCE layers: st->layer_ready_flags[0] is the source's [src num_layers] array (the other entries are
 * not read), and source layer l is read only once its flag reached st->epoch; layer_done_flags[l] (nullable, [src num_layers]) is
 * written once source layer l landed in every target that takes it; sync_workspace is u32[KVBM_SYNC_WORKSPACE_WORDS(src
 * num_layers)].  After the last byte, every target's done_flag and st->done_flag receive st->epoch, then completion_flag
 * receives completion_value: the completion word always comes last.  The spinning form is one persistent grid that claims (source
 * layer, big block, outer) units in layer-major order and waits once per source layer it enters; its last CTA writes every flag.
 * After a gate timeout no done flag is written (neither st->done_flag nor any target's) and completion_flag becomes 0xFFFFFFFF.
 * The stream-wait form waits on the stream once per source layer and launches the unstreamed scatter over that layer; the target
 * done flags are written after the last layer only.  The argument rules are kvbm_kernels_paged_repage_scatter's plus the gate's
 * with one source, all checked before any CUDA call.  An empty token or layer range waits for nothing and writes the done flags
 * and the completion word at once; it writes no layer_done_flags. */
cudaError_t kvbm_kernels_paged_repage_scatter_streamed(const kvbm_permute_side* src, uint32_t src_num_heads, uint32_t src_page_size,
                                                       const kvbm_scatter_target* targets, int num_targets, uint32_t dst_page_size,
                                                       uint32_t token_begin, uint32_t token_end, int layer_begin, int layer_end,
                                                       uint32_t src_row_bytes, int cast_mode, const float* cast_scales,
                                                       const kvbm_permute_stream* st, cudaStream_t stream);

/* kvbm_kernels_paged_repage_scatter over a batch of sequences: what a continuous-batching prefill step finishes at once, each
 * sequence with its own prefix-cache hit (token_begin, often inside a block), length and block tables, pushed to every target in
 * ONE launch.  Source, targets, windows, pages, layer range, formats, cast and scales are the launch's, as there; the token ranges
 * are `seqs` (host memory).  Concatenated tables: src->block_ids and every target's side.block_ids are concatenations in batch
 * order, sequence i contributing its table[token_begin / P .. ceil(token_end / P)) for that side's page P (nothing when its range
 * is empty).  Every target has Pd, so every target's concatenated table has the same per-sequence offsets, and the unit table of
 * kvbm_kernels_repage_batch_units(seqs, Ps, Pd) serves every target: `units` is device-accessible memory holding what it
 * produced, the caller's memory, read by the kernel and not on the host, valid until the launch has run.
 * Equivalence: a batch of one sequence writes exactly the bytes of kvbm_kernels_paged_repage_scatter with that range, and a batch
 * of n the bytes of n such launches in any order.  Two sequences may share SOURCE blocks (a shared prefix).  Within one target
 * pool, two sequences must not share a DESTINATION block: the entry cannot read device ids, so this is the caller's rule.
 * One signal for the batch: every target's done_flag and completion_flag are written once, after every sequence landed.
 * num_seqs == 0, only empty ranges, or an empty layer range move nothing and still signal.  cudaErrorInvalidValue, before any
 * CUDA call, for: every rule of kvbm_kernels_paged_repage_scatter but the token range's; any rule of
 * kvbm_kernels_repage_batch_units (a null seqs with num_seqs > 0 among them); a num_units other than the helper's count; a null
 * units with num_units > 0; num_units * layers * outer_dim of 2^31 or more. */
cudaError_t kvbm_kernels_paged_repage_scatter_batch(const kvbm_permute_side* src, uint32_t src_num_heads, uint32_t src_page_size,
                                                    const kvbm_scatter_target* targets, int num_targets, uint32_t dst_page_size,
                                                    const kvbm_repage_seq* seqs, size_t num_seqs, const kvbm_repage_unit* units,
                                                    size_t num_units, int layer_begin, int layer_end, uint32_t src_row_bytes,
                                                    int cast_mode, const float* cast_scales, uint32_t epoch, uint32_t* completion_flag,
                                                    uint32_t completion_value, cudaStream_t stream);

/* The batch streamed with kvbm_kernels_paged_repage_scatter_streamed's flag conventions.  A prefill batch computes layer l for
 * all its sequences together, so one ready flag per source layer covers the whole batch, and layer_done_flags[l] is written once
 * source layer l of EVERY sequence landed in every target that takes it.  After a gate timeout no done flag is written (neither
 * st->done_flag nor any target's) and completion_flag becomes 0xFFFFFFFF.  The stream-wait form launches the batch once per
 * source layer and writes the target done flags after the last layer only.  The argument rules are the batch's plus the gate's
 * with one source; a batch that moves nothing waits for nothing, writes the done flags and the completion word at once and no
 * layer_done_flags. */
cudaError_t kvbm_kernels_paged_repage_scatter_batch_streamed(const kvbm_permute_side* src, uint32_t src_num_heads, uint32_t src_page_size,
                                                             const kvbm_scatter_target* targets, int num_targets, uint32_t dst_page_size,
                                                             const kvbm_repage_seq* seqs, size_t num_seqs, const kvbm_repage_unit* units,
                                                             size_t num_units, int layer_begin, int layer_end, uint32_t src_row_bytes,
                                                             int cast_mode, const float* cast_scales, const kvbm_permute_stream* st,
                                                             cudaStream_t stream);

/* ---- the routed scatter: each sequence of a prefill batch to its own decode workers -------------------------------------------
 * A prefill batch mixes requests of several decode workers, so each sequence names the subset of the launch's targets it goes to:
 * targets, bit t = targets[t].  Host memory, as kvbm_repage_seq. */
typedef struct kvbm_route_seq {
  uint32_t token_begin, token_end, targets;
} kvbm_route_seq;

/* kvbm_repage_unit with the sequence's target mask in place of seq: a CTA loads its unit and its mask in one 16 B load. */
typedef struct kvbm_route_unit {
  uint32_t q0, tokens, small_k, targets;
} kvbm_route_unit;

/* Host-only (no GPU): kvbm_kernels_repage_batch_units over the ranges of seqs, with the same rules, counts and records, except
 * that each record's fourth word is its sequence's targets. */
int kvbm_kernels_repage_route_units(const kvbm_route_seq* seqs, size_t num_seqs, uint32_t src_page_size, uint32_t dst_page_size,
                                    kvbm_route_unit* out, size_t cap, size_t* num_units, size_t* src_ids, size_t* dst_ids);

/* kvbm_kernels_paged_repage_scatter_batch with a target mask per sequence, in ONE launch with one signal: for each sequence i, the
 * bytes of kvbm_kernels_paged_repage_scatter over i's range with only the targets whose bit is set in seqs[i].targets.  Every
 * other destination byte keeps its value, including the blocks of a target's table at the positions of sequences not routed to
 * it.  With every mask all num_targets bits, the bytes of kvbm_kernels_paged_repage_scatter_batch on the same inputs.
 * Tables: every target's concatenated table has the batch layout, sequence i contributing its table[token_begin / Pd ..
 * ceil(token_end / Pd)) whether or not it is routed to that target; entries of sequences not routed to a target are never read
 * and may hold any value, so one unit table, kvbm_kernels_repage_route_units(seqs, Ps, Pd), serves every target.  Only bits below
 * num_targets are ever consulted, on the host and in the kernel.  Within one target pool, two sequences routed to it must not
 * share a destination block.  Everything else is the batch scatter's: casts and scales, layer and head windows, shared source
 * blocks, the done flags and the completion word written once after every sequence landed.  cudaErrorInvalidValue, before any
 * CUDA call, for: every rule of kvbm_kernels_paged_repage_scatter_batch (with kvbm_kernels_repage_route_units for the unit
 * count), and a sequence whose targets is 0 or has a bit at or above num_targets. */
cudaError_t kvbm_kernels_paged_repage_scatter_routed(const kvbm_permute_side* src, uint32_t src_num_heads, uint32_t src_page_size,
                                                     const kvbm_scatter_target* targets, int num_targets, uint32_t dst_page_size,
                                                     const kvbm_route_seq* seqs, size_t num_seqs, const kvbm_route_unit* units,
                                                     size_t num_units, int layer_begin, int layer_end, uint32_t src_row_bytes,
                                                     int cast_mode, const float* cast_scales, uint32_t epoch, uint32_t* completion_flag,
                                                     uint32_t completion_value, cudaStream_t stream);

/* The routed scatter streamed with kvbm_kernels_paged_repage_scatter_batch_streamed's flag conventions: one ready flag per source
 * layer covers the batch, and layer_done_flags[l] is written once source layer l of every sequence landed in every target it is
 * routed to.  After a gate timeout no done flag is written and completion_flag becomes 0xFFFFFFFF.  The argument rules are the
 * routed scatter's plus the gate's with one source. */
cudaError_t kvbm_kernels_paged_repage_scatter_routed_streamed(const kvbm_permute_side* src, uint32_t src_num_heads, uint32_t src_page_size,
                                                              const kvbm_scatter_target* targets, int num_targets, uint32_t dst_page_size,
                                                              const kvbm_route_seq* seqs, size_t num_seqs, const kvbm_route_unit* units,
                                                              size_t num_units, int layer_begin, int layer_end, uint32_t src_row_bytes,
                                                              int cast_mode, const float* cast_scales, const kvbm_permute_stream* st,
                                                              cudaStream_t stream);

/* ---- the routed gather: each sequence of a decode step from the prefill workers that served it -------------------------------
 * The pull-side counterpart of the routed scatter, with the same kvbm_route_seq / kvbm_route_unit and
 * kvbm_kernels_repage_route_units: on the gather, bit s of a sequence's `targets` names srcs[s] (one kvbm_stage_source, one
 * window), the sources the sequence is read from.
 * kvbm_kernels_paged_stage_repage_gather_batch with a source mask per sequence, in ONE launch with one signal: for each sequence
 * i, the bytes of kvbm_kernels_paged_stage_repage_gather over i's range with only the windows whose bit is set in
 * seqs[i].targets.  Every other destination byte keeps its value (a layer none of i's windows covers included).  Tables: every
 * source's concatenated table has the batch layout, sequence i contributing its table whether or not it is routed to that
 * source; positions of sequences not routed to a source are never read and may hold any value, so one unit table,
 * kvbm_kernels_repage_route_units(seqs, Ps, Pd), serves every source.  A source no sequence is routed to is never read or
 * waited on.  One rule differs from the batch gather: two head windows of one stage may share destination heads when no
 * sequence's mask holds both (two prefill workers' windows write the same decode heads, for different sequences); the 256-head
 * limit counts every window's heads, shared or not.  Everything else is the batch gather's: stages, layer windows, casts and
 * scales, shared source blocks, no destination block in two sequences, and the done / completion flags written once after every
 * sequence landed.  cudaErrorInvalidValue, before any CUDA call, for: every rule of kvbm_kernels_paged_stage_repage_gather_batch
 * but the shared heads (with kvbm_kernels_repage_route_units for the unit count), a sequence whose mask is 0 or has a bit at or
 * above num_srcs, and a mask holding two windows of one stage that share a destination head. */
cudaError_t kvbm_kernels_paged_stage_repage_gather_routed(const kvbm_stage_source* srcs, int num_srcs, uint32_t src_page_size,
                                                          const kvbm_permute_side* dst, uint32_t dst_num_heads, uint32_t dst_page_size,
                                                          const kvbm_route_seq* seqs, size_t num_seqs, const kvbm_route_unit* units,
                                                          size_t num_units, int layer_begin, int layer_end, uint32_t src_row_bytes,
                                                          int cast_mode, const float* cast_scales, uint32_t* done_flag, uint32_t epoch,
                                                          uint32_t* completion_flag, uint32_t completion_value, cudaStream_t stream);

/* The routed gather streamed with kvbm_kernels_paged_stage_repage_gather_batch_streamed's flag conventions: one ready flag per
 * (source, layer) covers the batch, and layer_done_flags[l] is written once layer l of every sequence landed.  Only the sources
 * some sequence is routed to are waited on and need st->layer_ready_flags[s]; the others may be NULL.  The argument rules are
 * the routed gather's plus the gate's. */
cudaError_t kvbm_kernels_paged_stage_repage_gather_routed_streamed(const kvbm_stage_source* srcs, int num_srcs, uint32_t src_page_size,
                                                                   const kvbm_permute_side* dst, uint32_t dst_num_heads,
                                                                   uint32_t dst_page_size, const kvbm_route_seq* seqs, size_t num_seqs,
                                                                   const kvbm_route_unit* units, size_t num_units, int layer_begin,
                                                                   int layer_end, uint32_t src_row_bytes, int cast_mode,
                                                                   const float* cast_scales, const kvbm_permute_stream* st,
                                                                   cudaStream_t stream);

/* ---- re-paging between pages that need not divide: a batch gather and a batch scatter for any two page sizes ------------------
 * Engines configured independently keep pages that neither divide: a hybrid model's attention block of 544 tokens against a
 * decode engine's 64, or 24 against 16.  Every entry above rejects such a pair; the entries below take any two non-zero pages.
 * The unit stays one block of the larger-page side.  Its block's slot 0 is sequence position F = j * big_page; the smaller-page
 * side's block that holds F is entry small_k of its concatenated table, and F sits at slot `phase` = F % small_page of it.  The
 * token at big slot q then sits at offset phase + q from the start of that small block: in block small_k + (phase + q) /
 * small_page, slot (phase + q) % small_page.  With dividing pages every phase is 0.
 * Exactness bound: (big_page + small_page - gcd(big_page, small_page)) * small_page < 2^32.  phase + q stays below
 * big_page + small_page - gcd, and the kernels' multiply-high split by small_page is exact for it under this bound; with dividing
 * pages it is the other entries' big_page * small_page < 2^32.  As there, every sequence's last block of the larger page ends
 * below 2^32 tokens. */

/* kvbm_repage_unit with the block's phase in place of seq: a CTA loads its unit and its phase in one 16 B load.  q0, tokens and
 * small_k are kvbm_repage_unit's, small_k being the entry that holds the big block's slot 0 (wrapping below 0 as there); phase:
 * that slot 0's slot in small block small_k, below small_page. */
typedef struct kvbm_repage_anypage_unit {
  uint32_t q0, tokens, small_k, phase;
} kvbm_repage_anypage_unit;

/* Host-only (no GPU): kvbm_kernels_repage_batch_units for any two non-zero pages, with its conventions (sizing call, counts,
 * concatenated tables, the small_k wrap) and the records above.  For dividing pages its records and counts are that helper's
 * with phase 0 in place of seq.  Returns non-zero, writing nothing, for a null seqs with num_seqs > 0, a page of 0, pages past
 * the exactness bound, a reversed range, or a sequence whose last block of the larger page ends at or past 2^32 tokens. */
int kvbm_kernels_repage_anypage_units(const kvbm_repage_seq* seqs, size_t num_seqs, uint32_t src_page_size, uint32_t dst_page_size,
                                      kvbm_repage_anypage_unit* out, size_t cap, size_t* num_units, size_t* src_ids, size_t* dst_ids);

/* kvbm_kernels_paged_stage_repage_gather_batch for any two non-zero pages: the same parameters, with `units` the device-accessible
 * table kvbm_kernels_repage_anypage_units produced for the same seqs and pages.  Everything is the batch's: stages, layer and head
 * windows, casts and scales, shared source blocks, no destination block in two sequences, one signal after every sequence
 * landed, the empty batch's signal and the 2^31 unit bound.  A single range is a batch of one.  With dividing pages it writes
 * exactly the bytes of kvbm_kernels_paged_stage_repage_gather_batch.  When the destination has the smaller page, two units may
 * write disjoint token slots of one destination block.  cudaErrorInvalidValue, before any CUDA call, for every rule of
 * kvbm_kernels_paged_stage_repage_gather_batch but the divisibility of the pages, with kvbm_kernels_repage_anypage_units in place
 * of kvbm_kernels_repage_batch_units. */
cudaError_t kvbm_kernels_paged_stage_repage_gather_anypage(const kvbm_stage_source* srcs, int num_srcs, uint32_t src_page_size,
                                                           const kvbm_permute_side* dst, uint32_t dst_num_heads, uint32_t dst_page_size,
                                                           const kvbm_repage_seq* seqs, size_t num_seqs, const kvbm_repage_anypage_unit* units,
                                                           size_t num_units, int layer_begin, int layer_end, uint32_t src_row_bytes,
                                                           int cast_mode, const float* cast_scales, uint32_t* done_flag, uint32_t epoch,
                                                           uint32_t* completion_flag, uint32_t completion_value, cudaStream_t stream);

/* kvbm_kernels_paged_stage_repage_gather_anypage streamed with kvbm_kernels_paged_stage_repage_gather_batch_streamed's flag
 * conventions and gate forms; the stream-wait form launches the unstreamed anypage kernel per layer.  The argument rules are the
 * anypage gather's plus the gate's. */
cudaError_t kvbm_kernels_paged_stage_repage_gather_anypage_streamed(const kvbm_stage_source* srcs, int num_srcs, uint32_t src_page_size,
                                                                    const kvbm_permute_side* dst, uint32_t dst_num_heads,
                                                                    uint32_t dst_page_size, const kvbm_repage_seq* seqs, size_t num_seqs,
                                                                    const kvbm_repage_anypage_unit* units, size_t num_units, int layer_begin,
                                                                    int layer_end, uint32_t src_row_bytes, int cast_mode,
                                                                    const float* cast_scales, const kvbm_permute_stream* st,
                                                                    cudaStream_t stream);

/* kvbm_kernels_paged_repage_scatter_batch for any two non-zero pages: the push-side counterpart of the anypage gather, one source
 * of page Ps into up to KVBM_GATHER_MAX_SOURCES targets of page Pd in ONE launch, each vector read and cast once and stored to
 * every target.  The same parameters, with `units` the device-accessible table kvbm_kernels_repage_anypage_units(seqs, Ps, Pd)
 * produced; as in the batch scatter, every target shares Pd and the batch layout, so one unit table (and its phases) serves every
 * target.  Everything is the batch scatter's: windows, stages, formats, casts and scales, shared source blocks, no destination
 * block in two sequences of one target pool, every target's done_flag and completion_flag written once after every sequence
 * landed, the empty batch's signal and the 2^31 unit bound.  A single range is a batch of one.  With dividing pages it writes
 * exactly the bytes of kvbm_kernels_paged_repage_scatter_batch.  When Pd < Ps two units may write disjoint token slots of one
 * target block; when Ps < Pd several units read one source block.  cudaErrorInvalidValue, before any CUDA call, for every rule
 * of kvbm_kernels_paged_repage_scatter_batch but the divisibility of the pages, with kvbm_kernels_repage_anypage_units (and its
 * exactness bound) in place of kvbm_kernels_repage_batch_units. */
cudaError_t kvbm_kernels_paged_repage_scatter_anypage(const kvbm_permute_side* src, uint32_t src_num_heads, uint32_t src_page_size,
                                                      const kvbm_scatter_target* targets, int num_targets, uint32_t dst_page_size,
                                                      const kvbm_repage_seq* seqs, size_t num_seqs, const kvbm_repage_anypage_unit* units,
                                                      size_t num_units, int layer_begin, int layer_end, uint32_t src_row_bytes,
                                                      int cast_mode, const float* cast_scales, uint32_t epoch, uint32_t* completion_flag,
                                                      uint32_t completion_value, cudaStream_t stream);

/* kvbm_kernels_paged_repage_scatter_anypage streamed with kvbm_kernels_paged_repage_scatter_batch_streamed's flag conventions and
 * gate forms: one ready flag per source layer covers the batch, layer_done_flags[l] is written once source layer l of every
 * sequence landed in every target, and after a gate timeout no done flag is written and completion_flag becomes 0xFFFFFFFF.  The
 * stream-wait form launches the unstreamed anypage scatter per source layer.  The argument rules are the anypage scatter's plus
 * the gate's with one source. */
cudaError_t kvbm_kernels_paged_repage_scatter_anypage_streamed(const kvbm_permute_side* src, uint32_t src_num_heads, uint32_t src_page_size,
                                                               const kvbm_scatter_target* targets, int num_targets, uint32_t dst_page_size,
                                                               const kvbm_repage_seq* seqs, size_t num_seqs,
                                                               const kvbm_repage_anypage_unit* units, size_t num_units, int layer_begin,
                                                               int layer_end, uint32_t src_row_bytes, int cast_mode, const float* cast_scales,
                                                               const kvbm_permute_stream* st, cudaStream_t stream);

/* ---- routed re-paging between pages that need not divide: each sequence to or from its own workers, any two page sizes -------
 * A hybrid-attention prefill pool (544-token blocks) in front of several decode workers with 64-token pages mixes requests of
 * those workers in one batch: the routed entries' masks and the anypage entries' phases in one launch.  Both fit the one 16 B
 * record.  A kernel entry rejects mask bits at or above its rank count, at most KVBM_GATHER_MAX_SOURCES = 16, so a mask needs 16
 * bits; the phase is below the small page, and the exactness bound with big >= small >= gcd gives small^2 < 2^32, so
 * small <= 65535 and phase <= 65534 also need 16 bits. */

/* kvbm_route_unit for pages that need not divide: route = targets | phase << 16 (targets: the sequence's mask, below 2^16;
 * phase: kvbm_repage_anypage_unit's). */
typedef struct kvbm_route_anypage_unit {
  uint32_t q0, tokens, small_k, route;
} kvbm_route_anypage_unit;

/* Host-only (no GPU): kvbm_kernels_repage_anypage_units over the ranges of seqs, with the same rules, counts, sizing call and
 * small_k wrap, each record's fourth word packing its sequence's targets (low 16 bits) with its phase (high 16 bits).  For
 * dividing pages its records are kvbm_kernels_repage_route_units', byte for byte; route >> 16 is kvbm_kernels_repage_anypage_units'
 * phase and route & 0xFFFF the mask.  Returns non-zero, writing nothing, for every rule of kvbm_kernels_repage_anypage_units and a
 * mask with a bit at or above 16. */
int kvbm_kernels_repage_route_anypage_units(const kvbm_route_seq* seqs, size_t num_seqs, uint32_t src_page_size,
                                            uint32_t dst_page_size, kvbm_route_anypage_unit* out, size_t cap,
                                            size_t* num_units, size_t* src_ids, size_t* dst_ids);

/* kvbm_kernels_paged_repage_scatter_routed for any two non-zero pages: the same parameters, with `units` the device-accessible table
 * kvbm_kernels_repage_route_anypage_units(seqs, Ps, Pd) produced.  Every rule, flag convention and error order is the routed
 * scatter's (a sequence whose targets is 0 or has a bit at or above num_targets is rejected), except that the pages need only the
 * exactness bound.  Equivalences: with every mask all num_targets bits, the bytes of kvbm_kernels_paged_repage_scatter_anypage;
 * with dividing pages, the bytes of kvbm_kernels_paged_repage_scatter_routed; with one target per sequence, the bytes of one
 * kvbm_kernels_paged_repage_scatter_anypage launch per target over the sequences routed to it. */
cudaError_t kvbm_kernels_paged_repage_scatter_routed_anypage(const kvbm_permute_side* src, uint32_t src_num_heads, uint32_t src_page_size,
                                                             const kvbm_scatter_target* targets, int num_targets, uint32_t dst_page_size,
                                                             const kvbm_route_seq* seqs, size_t num_seqs, const kvbm_route_anypage_unit* units,
                                                             size_t num_units, int layer_begin, int layer_end, uint32_t src_row_bytes,
                                                             int cast_mode, const float* cast_scales, uint32_t epoch,
                                                             uint32_t* completion_flag, uint32_t completion_value, cudaStream_t stream);

/* kvbm_kernels_paged_repage_scatter_routed_anypage streamed with kvbm_kernels_paged_repage_scatter_routed_streamed's flag
 * conventions and gate forms: layer_done_flags[l] is written once source layer l of every sequence landed in every target it is
 * routed to, and after a gate timeout no done flag is written and completion_flag becomes 0xFFFFFFFF.  The stream-wait form
 * launches the unstreamed entry per source layer.  The argument rules are the unstreamed entry's plus the gate's with one source. */
cudaError_t kvbm_kernels_paged_repage_scatter_routed_anypage_streamed(const kvbm_permute_side* src, uint32_t src_num_heads,
                                                                      uint32_t src_page_size, const kvbm_scatter_target* targets,
                                                                      int num_targets, uint32_t dst_page_size, const kvbm_route_seq* seqs,
                                                                      size_t num_seqs, const kvbm_route_anypage_unit* units,
                                                                      size_t num_units, int layer_begin, int layer_end,
                                                                      uint32_t src_row_bytes, int cast_mode, const float* cast_scales,
                                                                      const kvbm_permute_stream* st, cudaStream_t stream);

/* kvbm_kernels_paged_stage_repage_gather_routed for any two non-zero pages: the same parameters, with `units` the
 * device-accessible table kvbm_kernels_repage_route_anypage_units(seqs, Ps, Pd) produced.  Every rule and error order is the
 * routed gather's (a mask of 0 or with a bit at or above num_srcs is rejected; two windows of one stage may share destination
 * heads when no mask holds both), except that the pages need only the exactness bound.  Equivalences: with every mask all
 * num_srcs bits, the bytes of kvbm_kernels_paged_stage_repage_gather_anypage; with dividing pages, the bytes of
 * kvbm_kernels_paged_stage_repage_gather_routed; with one source per sequence, the bytes of one
 * kvbm_kernels_paged_stage_repage_gather_anypage launch per source over the sequences routed to it. */
cudaError_t kvbm_kernels_paged_stage_repage_gather_routed_anypage(const kvbm_stage_source* srcs, int num_srcs, uint32_t src_page_size,
                                                                  const kvbm_permute_side* dst, uint32_t dst_num_heads,
                                                                  uint32_t dst_page_size, const kvbm_route_seq* seqs, size_t num_seqs,
                                                                  const kvbm_route_anypage_unit* units, size_t num_units, int layer_begin,
                                                                  int layer_end, uint32_t src_row_bytes, int cast_mode,
                                                                  const float* cast_scales, uint32_t* done_flag, uint32_t epoch,
                                                                  uint32_t* completion_flag, uint32_t completion_value, cudaStream_t stream);

/* kvbm_kernels_paged_stage_repage_gather_routed_anypage streamed with kvbm_kernels_paged_stage_repage_gather_routed_streamed's flag
 * conventions and gate forms: only the sources some sequence is routed to are waited on and need st->layer_ready_flags[s]; after a
 * gate timeout no done flag is written and completion_flag becomes 0xFFFFFFFF.  The stream-wait form launches the unstreamed entry
 * per layer.  The argument rules are the unstreamed entry's plus the gate's. */
cudaError_t kvbm_kernels_paged_stage_repage_gather_routed_anypage_streamed(const kvbm_stage_source* srcs, int num_srcs,
                                                                           uint32_t src_page_size, const kvbm_permute_side* dst,
                                                                           uint32_t dst_num_heads, uint32_t dst_page_size,
                                                                           const kvbm_route_seq* seqs, size_t num_seqs,
                                                                           const kvbm_route_anypage_unit* units, size_t num_units,
                                                                           int layer_begin, int layer_end, uint32_t src_row_bytes,
                                                                           int cast_mode, const float* cast_scales,
                                                                           const kvbm_permute_stream* st, cudaStream_t stream);

/* Host-only (no GPU): the stride table kvbm_kernels_paged_permute walks with for one side.  out[0] = 1 when offsets count
 * from the block's first byte (universal formats) or 0 when they count from the (layer, outer) region's first byte; the
 * element (layer l, outer o, head h, token t) then sits at  [out[0] ? l * out[1] + o * out[2] : 0] + h * out[3] + t * out[4].
 * Returns non-zero for formats without a kernel or strides that are not multiples of 16. */
int kvbm_kernels_permute_strides(int kv_layout, uint32_t num_layers, uint32_t outer_dim, uint32_t num_heads, uint32_t page_size,
                                 uint32_t row_bytes, uint64_t block_stride, uint64_t outer_stride, uint64_t out[5]);

/* 1 when KVBM_GATE_AUTO would let the transfer's warps spin on the ready flags (eager module loading detected through
 * cuModuleGetLoadingMode), 0 when it would gate on the stream instead. */
int kvbm_kernels_gate_would_spin(void);

/* Small helpers so hosts without a CUDA binding (ctypes, cgo, JNI) can drive the flags.  wait_flag holds the stream until
 * (int32_t)(*flag - value) >= 0, the epoch order of kvbm_paged_copy_opts.epoch. */
cudaError_t kvbm_kernels_set_flags(uint32_t* flags, int first, int count, uint32_t value,
                                   cudaStream_t stream);
cudaError_t kvbm_kernels_wait_flag(const uint32_t* flag, uint32_t value, cudaStream_t stream);
/* cudaStreamWaitEvent for hosts without a CUDA binding: `event` is a raw cudaEvent_t / CUevent handle.  With
 * set_flags this turns an engine's existing per-layer event into a device-side ready flag on a helper stream. */
cudaError_t kvbm_kernels_stream_wait_event(cudaStream_t stream, void* event);

/* Number of kernel launches issued by this library since load (bench accounting). */
uint64_t kvbm_kernels_launch_count(void);
/* "sm_90a" build tag + whether the TMA path is compiled in. */
const char* kvbm_kernels_build_info(void);

#ifdef __cplusplus
}
#endif
#endif /* KVBM_KERNELS_H */
