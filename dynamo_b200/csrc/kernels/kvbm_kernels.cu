// libkvbm_kernels.so -- sm_90a KV-block transfer kernels behind the reference C ABI
// (see include/kvbm_kernels.h for the contract and the reference lines each entry replaces).
#include <cuda_runtime_api.h>

#include "../../../include/kvbm_kernels.h"
#include "copy_engine.cuh"

#include <algorithm>
#include <atomic>
#include <mutex>
#include <numeric>
#include <type_traits>
#include <cstdio>
#include <vector>

static bool eager_module_loading();

namespace kvbm {

// ------------------------------------------------------------------------------------------------
// launch bookkeeping
// ------------------------------------------------------------------------------------------------
static std::atomic<uint64_t> g_launches{0};

struct DeviceInfo {
  int sm_count = 0;
  int max_smem_optin = 0;
};

static cudaError_t preload_kernels();

static cudaError_t device_info(DeviceInfo* out)
{
  constexpr int kMaxDev = 64;
  static std::atomic<int> sm[kMaxDev];
  static std::atomic<int> smem[kMaxDev];
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  if (dev < 0 || dev >= kMaxDev) return cudaErrorInvalidDevice;
  int s = sm[dev].load(std::memory_order_acquire);
  if (s == 0) {
    int a = 0, b = 0;
    if ((e = cudaDeviceGetAttribute(&a, cudaDevAttrMultiProcessorCount, dev)) != cudaSuccess) return e;
    if ((e = cudaDeviceGetAttribute(&b, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev)) != cudaSuccess) return e;
    // CUDA loads kernels lazily and a first-time load can wait for the device to go idle.  A transfer kernel
    // that is spinning on layer-ready flags would then deadlock against the very first launch of the tiny
    // flag kernel that is supposed to release it -- so every kernel of this library is loaded up front.
    if ((e = preload_kernels()) != cudaSuccess) return e;
    smem[dev].store(b, std::memory_order_release);
    sm[dev].store(a, std::memory_order_release);
    s = a;
  }
  out->sm_count = s;
  out->max_smem_optin = smem[dev].load(std::memory_order_acquire);
  return cudaSuccess;
}

static int default_ctas(const DeviceInfo& di) { return di.sm_count; }

// Ring geometry of one launch.
struct RingCfg {
  int rings;        // R rings per CTA (2 warps each)
  int stages;       // S (input slots per ring)
  int pending;      // P (TMA stores allowed to keep draining their slot); loads ahead = S - P
  int batch;        // largest scheduler ticket, items
  uint32_t tile;    // source bytes per slot
  uint32_t smem;    // dynamic shared memory bytes
  uint32_t out_tile;  // cast only
};

// Defaults.  One SM moves a bounded number of bytes per second through the TMA however many rings it runs, so the
// HBM-bound copy wants every SM: one CTA per SM (132 on an H100 SXM).  A whole 32 KiB region per bulk op keeps the
// per-item instruction chain short; smaller regions get more rings per CTA instead (~192 KiB of slots per CTA either
// way, within the 227 KiB a block may opt into on sm_90).  Callers that overlap the transfer with compute and need
// only NVLink peer bandwidth pass max_ctas.  benchmarks/copylab.cu sweeps these choices.
constexpr int kDefaultStages = 6;
constexpr uint32_t kDefaultTile = 32768;
constexpr int kDefaultBatch = 8;

static uint32_t round_up(uint32_t x, uint32_t m) { return (x + m - 1) / m * m; }

// cast: 0 none, 1 up (out = 2x), 2 down (out = x/2).  `warps` is the legacy knob: 2 warps make one ring.
static RingCfg make_ring(const DeviceInfo& di, uint32_t unit_bytes, int warps, int stages, int tile, int cast, int pending = 0)
{
  RingCfg c{};
  c.batch = kDefaultBatch;
  // default tile: the whole unit when it is small, else kDefaultTile pieces
  uint32_t t = tile > 0 ? static_cast<uint32_t>(tile) : std::min<uint32_t>(std::max<uint32_t>(unit_bytes, 16), kDefaultTile);
  t = round_up(t, 32);
  // rings per CTA: as many as keep ~32 KiB x S of slots busy (1 for 32 KiB tiles, 2 for 16 KiB, 4 for <= 8 KiB)
  c.rings = warps > 0 ? std::max(1, std::min(warps, 16) / 2) : static_cast<int>(std::max<uint32_t>(1, std::min<uint32_t>(4, kDefaultTile / t)));
  const uint32_t budget = static_cast<uint32_t>(di.max_smem_optin) - 1024;
  for (;;) {
    const uint32_t out = cast == 1 ? 2 * t : (cast == 2 ? t / 2 : 0);
    // default depth: ~96 KiB of slots per ring (small tiles get more slots), at least 3, at most 12
    int s = stages > 0 ? stages : kDefaultStages;
    s = std::max(2, std::min(s, kMaxStages));  // one slot cannot overlap a load with a store
    while (s > 2 && cta_smem_bytes(c.rings, s, t, out) > budget) --s;
    if (cta_smem_bytes(c.rings, s, t, out) <= budget) {
      c.stages = s;
      c.pending = pending > 0 ? std::min(pending, s - 1) : std::max(1, s / 3);  // 2 of 6
      c.tile = t;
      c.out_tile = out;
      c.smem = cta_smem_bytes(c.rings, s, t, out);
      return c;
    }
    if (t > 1024)
      t = round_up(t / 2, 32);
    else if (c.rings > 1)
      c.rings /= 2;
    else {
      c.stages = 2;
      c.pending = 1;
      c.tile = t;
      c.out_tile = out;
      c.smem = cta_smem_bytes(1, 2, t, out);
      return c;
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Scheduler words for launches that bring no workspace (legacy callers, opts == NULL): a small per-device pool of
// zeroed 4-word slots.  A slot is handed to one launch at a time: an event recorded behind the launch tells when it
// may be reused (the kernel leaves the words zeroed).  No free slot, or a stream that is being captured into a
// graph, simply means a static tile schedule for that launch -- never a wait.
// ------------------------------------------------------------------------------------------------
struct SchedPool {
  static constexpr int kSlots = 64;
  std::mutex mu;
  uint32_t* words = nullptr;  // kSlots * 4
  cudaEvent_t ev[kSlots] = {};
  bool used[kSlots] = {};
  int next = 0;
  bool failed = false;
};
static SchedPool g_pools[64];

static uint32_t* sched_acquire(int dev, cudaStream_t stream, int* slot_out)
{
  *slot_out = -1;
  cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
  if (cudaStreamIsCapturing(stream, &cap) != cudaSuccess || cap != cudaStreamCaptureStatusNone) {
    (void)cudaGetLastError();
    return nullptr;
  }
  SchedPool& p = g_pools[dev];
  std::lock_guard<std::mutex> lk(p.mu);
  if (p.failed) return nullptr;
  if (!p.words) {
    if (cudaMalloc(&p.words, SchedPool::kSlots * 16) != cudaSuccess || cudaMemset(p.words, 0, SchedPool::kSlots * 16) != cudaSuccess) {
      (void)cudaGetLastError();
      p.failed = true;
      p.words = nullptr;
      return nullptr;
    }
    for (int i = 0; i < SchedPool::kSlots; ++i)
      if (cudaEventCreateWithFlags(&p.ev[i], cudaEventDisableTiming) != cudaSuccess) {
        (void)cudaGetLastError();
        p.failed = true;
        return nullptr;
      }
  }
  for (int n = 0; n < SchedPool::kSlots; ++n) {
    const int i = (p.next + n) % SchedPool::kSlots;
    if (p.used[i]) {
      if (cudaEventQuery(p.ev[i]) != cudaSuccess) {
        (void)cudaGetLastError();
        continue;
      }
      p.used[i] = false;
    }
    p.used[i] = true;  // busy until sched_release records its event (and that event completes)
    p.next = (i + 1) % SchedPool::kSlots;
    *slot_out = i;
    return p.words + 4 * i;
  }
  return nullptr;
}

static void sched_release(int dev, int slot, cudaStream_t stream)
{
  if (slot < 0) return;
  SchedPool& p = g_pools[dev];
  std::lock_guard<std::mutex> lk(p.mu);
  if (cudaEventRecord(p.ev[slot], stream) != cudaSuccess) {
    (void)cudaGetLastError();
    // cannot tell when the launch ends: retire the slot for good rather than risk sharing it
  }
}

// ------------------------------------------------------------------------------------------------
// K1: pointer-pair copy (legacy ABI).  Hardware-scheduled SIMT: one CTA per (pair, 32 KiB chunk) -- or one warp per
// pair when pairs are small -- 4 independent 16 B loads in flight per thread (8 and 4 are equal on HBM, 4 is a little
// better when the source is pinned host memory), the alignment ladder of the reference.
// The CTA scheduler is the dynamic load balancer here, so the ABI needs no workspace and the library no state.
// ------------------------------------------------------------------------------------------------
constexpr uint32_t kPairChunk = 32768;
constexpr uint32_t kPairSmall = 4096;
constexpr int kPairThreads = 256;
constexpr int kPairLoads = 4;

__global__ void __launch_bounds__(kPairThreads)
kvbm_pair_copy_kernel(void* const* __restrict__ src_ptrs, void* const* __restrict__ dst_ptrs, size_t copy_size,
                      uint32_t chunks_per_pair, uint64_t num_pairs)
{
  const uint64_t bid = blockIdx.x + static_cast<uint64_t>(gridDim.x) * blockIdx.y;
  if (copy_size <= kPairSmall) {  // warp per pair
    const uint64_t pair = bid * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (pair >= num_pairs) return;
    group_copy_simt<kPairLoads>(static_cast<uint8_t*>(dst_ptrs[pair]), static_cast<const uint8_t*>(src_ptrs[pair]), copy_size, threadIdx.x & 31, 32);
    return;
  }
  const uint64_t pair = bid / chunks_per_pair;
  if (pair >= num_pairs) return;
  const uint32_t chunk = static_cast<uint32_t>(bid - pair * chunks_per_pair);
  const size_t off = static_cast<size_t>(chunk) * kPairChunk;
  const size_t left = copy_size - off;
  // chunk boundaries are multiples of 32 KiB, so the alignment class of (src, dst) is the same for every chunk
  group_copy_simt<kPairLoads>(static_cast<uint8_t*>(dst_ptrs[pair]) + off, static_cast<const uint8_t*>(src_ptrs[pair]) + off,
                              left < kPairChunk ? left : kPairChunk, threadIdx.x, blockDim.x);
}

// ------------------------------------------------------------------------------------------------
// v2: block-table (paged) gather -> push -> scatter, addresses computed on the device
// ------------------------------------------------------------------------------------------------
struct PagedArgs {
  kvbm_paged_layout src;
  kvbm_paged_layout dst[kMaxDst];
  const int32_t* src_ids[kMaxDst];
  const int32_t* dst_ids[kMaxDst];
  int ndst;        // destinations
  int replicate;   // 1: all destinations share src_ids[0] -> read once, store ndst times
  uint32_t n_blocks;
  uint32_t layer_begin, n_layers;  // layers [layer_begin, layer_begin + n_layers)
  uint32_t outer;
  uint32_t tiles_per_region;
  uint32_t tile;      // source bytes per piece
  uint32_t dst_num, dst_den;  // destination bytes = source bytes * dst_num / dst_den (cast)
};

// PACK_OUTER (a scaled cast): Piece::layer = layer | o << 16, so the consumer can find the (layer, outer) scale (CastScales).
template <bool PACK_OUTER>
struct PagedGen {
  PagedArgs a;
  // item order (layer-major so a layer completes early for streaming):
  //   item = (((layer * n_blocks + block) * outer + o) * fan + d) * tiles_per_region + t
  // where fan = ndst for distinct payloads (destinations interleaved -> all NVLink ports busy) and 1
  // when replicating.
  __device__ __forceinline__ void get(uint32_t item, Piece& p) const
  {
    uint32_t r = item / a.tiles_per_region;
    const uint32_t t = item - r * a.tiles_per_region;
    uint32_t d = 0;
    if (!a.replicate) {
      const uint32_t r2 = r / a.ndst;
      d = r - r2 * a.ndst;
      r = r2;
    }
    uint32_t r2 = r / a.outer;
    const uint32_t o = r - r2 * a.outer;
    r = r2;
    r2 = r / a.n_blocks;
    const uint32_t blk = r - r2 * a.n_blocks;
    const uint32_t layer = a.layer_begin + r2;

    const uint64_t soff = static_cast<uint64_t>(t) * a.tile;
    const uint32_t left = a.src.region_bytes - static_cast<uint32_t>(soff);
    p.bytes = left < a.tile ? left : a.tile;
    p.layer = PACK_OUTER ? static_cast<int>(layer | (o << 16)) : static_cast<int>(layer);
    const uint64_t doff = soff * a.dst_num / a.dst_den;
    const int32_t sb = __ldg(a.src_ids[d] + blk);
    p.src = reinterpret_cast<const uint8_t*>(__ldg(a.src.layer_base + layer) + static_cast<uint64_t>(sb) * a.src.block_stride +
                                             static_cast<uint64_t>(o) * a.src.outer_stride + soff);
    if (a.replicate) {
      p.ndst = a.ndst;
#pragma unroll
      for (int k = 0; k < kMaxDst; ++k) {
        if (k < a.ndst) {
          const int32_t db = __ldg(a.dst_ids[k] + blk);
          p.dst[k] = reinterpret_cast<uint8_t*>(__ldg(a.dst[k].layer_base + layer) +
                                                static_cast<uint64_t>(db) * a.dst[k].block_stride +
                                                static_cast<uint64_t>(o) * a.dst[k].outer_stride + doff);
        }
      }
    } else {
      p.ndst = 1;
      const int32_t db = __ldg(a.dst_ids[d] + blk);
      // select destination d without dynamic indexing of a kernel-parameter array of structs
      const uint64_t* lb = a.dst[0].layer_base;
      uint64_t bs = a.dst[0].block_stride, os = a.dst[0].outer_stride;
#pragma unroll
      for (int k = 1; k < kMaxDst; ++k)
        if (k == static_cast<int>(d)) {
          lb = a.dst[k].layer_base;
          bs = a.dst[k].block_stride;
          os = a.dst[k].outer_stride;
        }
      p.dst[0] = reinterpret_cast<uint8_t*>(__ldg(lb + layer) + static_cast<uint64_t>(db) * bs +
                                            static_cast<uint64_t>(o) * os + doff);
    }
  }
};

struct PagedSyncArgs {
  const uint32_t* layer_ready;
  uint32_t* layer_counters;  // [num_layers] (user workspace) or null
  uint32_t* ctl;             // 3 control words: rings finished, abort, scheduler tickets; null = static schedule
  uint32_t* done_flag[kMaxDst];
  uint32_t* layer_done[kMaxDst];
  uint32_t* completion_flag;
  uint32_t completion_value;
  uint32_t epoch;
  uint64_t gate_timeout_ns;
  int num_flag_dsts;  // destinations that get flags (== data destinations unless multicast)
};

__device__ __forceinline__ StreamSync make_sync(const PagedSyncArgs& s, const PagedArgs& a, uint32_t total, int R)
{
  StreamSync ss{};
  ss.gate = s.layer_ready != nullptr;
  ss.want_layers = false;
  ss.want_done = s.completion_flag != nullptr;
  ss.layer_ready = s.layer_ready;
  ss.layer_counters = s.layer_counters;
  ss.ctl = s.ctl;
  ss.epoch = s.epoch;
  ss.gate_timeout_ns = s.gate_timeout_ns;
  ss.completion_flag = s.completion_flag;
  ss.completion_value = s.completion_value;
  ss.total_rings = gridDim.x * R;
  ss.items_per_layer = total / a.n_layers;
  ss.ndst = s.num_flag_dsts;
  ss.layer_begin = static_cast<int>(a.layer_begin);
  ss.layer_end = static_cast<int>(a.layer_begin + a.n_layers);
#pragma unroll
  for (int d = 0; d < kMaxDst; ++d) {
    ss.done_flag[d] = s.done_flag[d];
    ss.layer_done[d] = s.layer_done[d];
    if (d < s.num_flag_dsts && s.layer_done[d] != nullptr) ss.want_layers = true;
    if (d < s.num_flag_dsts && s.done_flag[d] != nullptr) ss.want_done = true;
  }
  if (ss.layer_counters == nullptr) ss.want_layers = false;
  return ss;
}

// SCALED: the cast applies scales[layer * outer + o] (kvbm_paged_copy_opts.cast_scales); only with a cast, never FAST.
template <int CAST, bool FAST, bool SCALED = false>
__global__ void __launch_bounds__(512, 1)
kvbm_paged_copy_kernel(const __grid_constant__ PagedGen<SCALED> gen, const __grid_constant__ PagedSyncArgs sync,
                       uint32_t total, int S, int P, int batch, int static_schedule, uint32_t out_tile, int allow_tma, int cache_hint,
                       int variant, const float* scales)
{
  extern __shared__ __align__(128) uint8_t smem[];
  const int R = blockDim.x >> 6;
  const int ring_ndst = gen.a.replicate ? gen.a.ndst : 1;
  const StreamSync ss = make_sync(sync, gen.a, total, R);
  RingParams rp{S, P, batch, gen.a.tile, out_tile, allow_tma != 0, static_schedule != 0, cache_hint, CAST == KVBM_CAST_NONE ? variant : 0};
  run_rings<CAST, FAST, SCALED>(smem, gen, total, ring_ndst, rp, ss, CastScales{scales, gen.a.outer});
}

// ------------------------------------------------------------------------------------------------
// K2 / K3: block stacks <-> universal, generic path for rows the head-row walk below does not take (not a whole number of
// 16-byte vectors, or past its bounds).  Index peel identical in meaning to the reference (tensor_kernels.cu:150-228) but
// done per VEC-byte vector when a head row allows it, and with 32-bit arithmetic; one thread moves VEC bytes.
// ------------------------------------------------------------------------------------------------
template <int VEC, bool TO_UNIVERSAL>
__global__ void __launch_bounds__(256)
kvbm_permute_kernel(void* const* universal_ptrs, void* const* block_ptrs, uint64_t total_units,
                    uint32_t units_per_block, uint32_t nh, uint32_t nl, uint32_t no, uint32_t nt,
                    uint32_t hdv /* row length in VEC units */, int layout)
{
  const uint64_t stride = static_cast<uint64_t>(blockDim.x) * gridDim.x;
  for (uint64_t u = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x; u < total_units; u += stride) {
    const uint32_t b = static_cast<uint32_t>(u / units_per_block);
    const uint32_t residual = static_cast<uint32_t>(u - static_cast<uint64_t>(b) * units_per_block);
    uint32_t tmp = residual;
    const uint32_t hd_i = tmp % hdv;
    tmp /= hdv;
    const uint32_t nt_i = tmp % nt;
    tmp /= nt;
    const uint32_t no_i = tmp % no;
    tmp /= no;
    const uint32_t nl_i = tmp % nl;
    const uint32_t nh_i = tmp / nl;
    const uint32_t chunk_off = layout == KVBM_BLOCK_LAYOUT_NHD ? ((nt_i * nh) + nh_i) * hdv + hd_i
                                                               : ((nh_i * nt) + nt_i) * hdv + hd_i;
    uint8_t* chunk = static_cast<uint8_t*>(block_ptrs[static_cast<size_t>(b) * nl * no + nl_i * no + no_i]) +
                     static_cast<size_t>(chunk_off) * VEC;
    uint8_t* uni = static_cast<uint8_t*>(universal_ptrs[b]) + static_cast<size_t>(residual) * VEC;
    uint8_t* d = TO_UNIVERSAL ? uni : chunk;
    const uint8_t* s = TO_UNIVERSAL ? chunk : uni;
    const bool aligned = ((reinterpret_cast<uintptr_t>(d) | reinterpret_cast<uintptr_t>(s)) & (VEC - 1)) == 0;
    if (!aligned) {
      // buffers only promise element alignment (>= 2 B): move the unit as 16-bit pieces
#pragma unroll
      for (int k = 0; k < VEC / 2; ++k)
        reinterpret_cast<uint16_t*>(d)[k] = reinterpret_cast<const uint16_t*>(s)[k];
    } else if (VEC == 16)
      *reinterpret_cast<uint4*>(d) = *reinterpret_cast<const uint4*>(s);
    else if (VEC == 8)
      *reinterpret_cast<uint2*>(d) = *reinterpret_cast<const uint2*>(s);
    else if (VEC == 4)
      *reinterpret_cast<uint32_t*>(d) = *reinterpret_cast<const uint32_t*>(s);
    else
      *reinterpret_cast<uint16_t*>(d) = *reinterpret_cast<const uint16_t*>(s);
  }
}

// ------------------------------------------------------------------------------------------------
// The head-row walk of the permuting kernels (K2 / K3 on pointer tables, and the paged transform).  For a fixed
// (block, layer, outer, head) the nt rows of one head sit at  base + head * head_stride + t * tok_stride  on either side,
// for every KvBlockLayout (kv_block_layout.rs:85-95):
//   UniversalTP [nh,nl,no,nt,hd]  base = block + (l*no + o)*nt*row     head_stride = nl*no*nt*row  tok_stride = row
//   UniversalPP [nl,nh,no,nt,hd]  base = block + l*nh*no*nt*row + o*nt*row   head_stride = no*nt*row   tok_stride = row
//   OperationalHND [nl,no,nh,nt,hd]  base = region(l, o)               head_stride = nt*row        tok_stride = row
//   OperationalNHD [nl,no,nt,nh,hd]  base = region(l, o)               head_stride = row           tok_stride = nh*row
// K2 / K3's chunk [nt,nh,hd] / [nh,nt,hd] is an OperationalNHD / HND region and its universal block is UniversalTP.
// One CTA per (block, layer, outer) unit -- the hardware CTA scheduler balances the SMs --, one warp per head, a few
// integer ops per 16 B vector (the reference peels 5 div/mod per ELEMENT, tensor_kernels.cu:150-187) and 8 independent
// 16 B loads per lane in flight before the first store.
// ------------------------------------------------------------------------------------------------
struct PermuteSide {
  const uint64_t* layer_base;
  const int32_t* ids;
  uint64_t block_stride;
  uint64_t layer_step;   // added per layer on top of layer_base[universal ? 0 : l]
  uint64_t outer_step;
  uint64_t head_stride;
  uint64_t tok_stride;
  int universal;
};

// The stride table above, for one side of a transform.  False for a format without one, or strides that are not whole
// 16 B vectors.
static bool fill_permute_side(const kvbm_permute_side& in, uint32_t nl, uint32_t no, uint32_t nh, uint32_t nt, uint32_t row, PermuteSide* out)
{
  const uint64_t head_run = static_cast<uint64_t>(nt) * row;
  PermuteSide p{};
  p.layer_base = in.layout.layer_base;
  p.ids = in.block_ids;
  p.block_stride = in.layout.block_stride;
  switch (in.kv_layout) {
    case KVBM_KV_UNIVERSAL_TP:
      p.universal = 1;
      p.layer_step = no * head_run;
      p.outer_step = head_run;
      p.head_stride = static_cast<uint64_t>(nl) * no * head_run;
      p.tok_stride = row;
      break;
    case KVBM_KV_UNIVERSAL_PP:
      p.universal = 1;
      p.layer_step = static_cast<uint64_t>(nh) * no * head_run;
      p.outer_step = head_run;
      p.head_stride = no * head_run;
      p.tok_stride = row;
      break;
    case KVBM_KV_OPERATIONAL_HND:
      p.outer_step = in.layout.outer_stride;
      p.head_stride = head_run;
      p.tok_stride = row;
      break;
    case KVBM_KV_OPERATIONAL_NHD:
      p.outer_step = in.layout.outer_stride;
      p.head_stride = row;
      p.tok_stride = static_cast<uint64_t>(nh) * row;
      break;
    default:
      return false;
  }
  if ((p.block_stride | p.outer_step) & 15) return false;
  *out = p;
  return true;
}

// How vector v of one head's run of nt rows splits into (token t, 16 B column c), v = t * V + c with V vectors per row:
// a shift and a mask when V is a power of two, else a multiply-high by ceil(2^32 / V) (head_dim 80, 96, 192, MLA's
// 576 ...), exact for v < 2^32 / V, so the 8 loads of a lane stay independent.
struct RowSplit {
  uint32_t vpr;    // pow2: log2 of V, else V
  uint32_t magic;  // !pow2: ceil(2^32 / V)
  bool pow2;
};

// The walk takes rows of a whole number of 16 B vectors, 16 B ... 64 KiB, and with the multiply-high only while
// nt * V < 2^32 / V.  False otherwise.
static bool row_split(uint64_t row_bytes, uint64_t nt, RowSplit* out)
{
  if (row_bytes < 16 || row_bytes > 65536 || (row_bytes & 15)) return false;
  const uint32_t V = static_cast<uint32_t>(row_bytes >> 4);
  if ((V & (V - 1)) == 0) {
    uint32_t log2_v = 0;
    while ((1u << log2_v) < V) ++log2_v;
    *out = {log2_v, 0u, true};
    return true;
  }
  if (nt * V >= (1ull << 32) / V) return false;
  *out = {V, static_cast<uint32_t>(((1ull << 32) + V - 1) / V), false};
  return true;
}

template <bool POW2>
__device__ __forceinline__ uint32_t row_run(const RowSplit& r, uint32_t nt)  // 16 B vectors of one head
{
  return POW2 ? nt << r.vpr : nt * r.vpr;
}

// Offset of vector v from its head's base, for a side whose vector is 2^SHIFT bytes (16, or 32 for the bf16 side of a
// cast).  32-bit: a head's rows lie within one region of nt * nh * row < 2^32 bytes.
template <bool POW2, int SHIFT = 4>
__device__ __forceinline__ uint32_t row_offset(const RowSplit& r, uint32_t v, uint32_t tok_stride)
{
  const uint32_t t = POW2 ? v >> r.vpr : __umulhi(v, r.magic);
  const uint32_t c = POW2 ? v & ((1u << r.vpr) - 1) : v - t * r.vpr;
  return t * tok_stride + (c << SHIFT);
}

// One unit: heads h0, h0 + hstep, ... < nh of it, one warp per head (h0 = the warp, hstep = the CTA's warps when a CTA
// walks one unit).  sb / db: the unit's bases; both must be 16 B aligned.  The last batch of
// a head is predicated rather than a serial tail: for head_dim 64 ... 96 in bf16 it is the whole head, and its loads stay
// independent.  With a cast (KVBM_CAST_*) the walk counts 16 B vectors of the fp8 side's row: one vector is 16 elements,
// 16 B on the fp8 side and 32 B on the bf16 side, so fp8 -> bf16 turns one load into two stores and bf16 -> fp8 two loads
// into one store.  Every lane keeps 8 independent 16 B loads in flight in all three forms.  SCALED: the cast applies `scale`,
// the fp8 side's dequantisation scale of the unit (one (block, layer, outer), so one scale).
template <int CAST, bool POW2, bool SCALED = false>
__device__ __forceinline__ void walk_head_rows(const uint8_t* sb, uint64_t s_head, uint32_t s_tok, uint8_t* db, uint64_t d_head,
                                               uint32_t d_tok, uint32_t h0, uint32_t hstep, uint32_t nh, uint32_t nt, const RowSplit& r,
                                               const ptx::Scale& scale = ptx::Scale{1.f, 1.f})
{
  constexpr int IN = CAST == KVBM_CAST_BF16_TO_FP8E4M3 ? 2 : 1;   // 16 B loads per vector
  constexpr int OUT = CAST == KVBM_CAST_FP8E4M3_TO_BF16 ? 2 : 1;  // 16 B stores per vector
  constexpr int U = 8 / IN;
  const uint32_t run = row_run<POW2>(r, nt);
  const int lane = threadIdx.x & 31;
  for (uint32_t h = h0; h < nh; h += hstep) {
    const uint8_t* sh = sb + h * s_head;
    uint8_t* dh = db + h * d_head;
    for (uint32_t v = lane; v < run; v += U * 32) {
      uint4 x[U][IN];
#pragma unroll
      for (int k = 0; k < U; ++k)
        if (v + k * 32 < run) {
          const uint8_t* s = sh + row_offset<POW2, 3 + IN>(r, v + k * 32, s_tok);
#pragma unroll
          for (int i = 0; i < IN; ++i) x[k][i] = ptx::ld_stream_v4(s + 16 * i);
        }
#pragma unroll
      for (int k = 0; k < U; ++k)
        if (v + k * 32 < run) {
          uint8_t* d = dh + row_offset<POW2, 3 + OUT>(r, v + k * 32, d_tok);
          if constexpr (CAST == KVBM_CAST_NONE) {
            ptx::st_stream_v4(d, x[k][0]);
          } else {
            uint4 y[OUT];
            cast_vector<SCALED>(x[k], y, scale);  // bit for bit the paged copy's cast rings (copy_engine.cuh)
#pragma unroll
            for (int i = 0; i < OUT; ++i) ptx::st_stream_v4(d + 16 * i, y[i]);
          }
        }
    }
  }
}

// K2 / K3 on the reference's pointer tables.  S is the source side, D the destination; the universal side's base is
// universal_ptrs[b] + l * layer_step + o * outer_step, the chunk side's is block_ptrs[unit].  The ABI only promises
// element alignment for the tables, so a unit whose bases are not 16 B aligned takes the same walk one element at a time.
template <bool POW2>
__global__ void __launch_bounds__(256)
kvbm_permute_table_kernel(void* const* __restrict__ universal_ptrs, void* const* __restrict__ block_ptrs, const __grid_constant__ PermuteSide S,
                          const __grid_constant__ PermuteSide D, uint32_t nl, uint32_t no, uint32_t nh, uint32_t nt, RowSplit r, uint32_t elem)
{
  const uint32_t unit = blockIdx.x;  // (b * nl + l) * no + o
  const uint32_t b = unit / (nl * no);
  const uint32_t rem = unit - b * (nl * no);
  const uint32_t l = rem / no, o = rem - l * no;
  auto base_of = [&](const PermuteSide& X) {
    return X.universal ? static_cast<uint8_t*>(universal_ptrs[b]) + l * X.layer_step + o * X.outer_step : static_cast<uint8_t*>(block_ptrs[unit]);
  };
  const uint8_t* sb = base_of(S);
  uint8_t* db = base_of(D);
  if (((reinterpret_cast<uintptr_t>(sb) | reinterpret_cast<uintptr_t>(db)) & 15) == 0) {
    walk_head_rows<KVBM_CAST_NONE, POW2>(sb, S.head_stride, S.tok_stride, db, D.head_stride, D.tok_stride, threadIdx.x >> 5, blockDim.x >> 5,
                                         nh, nt, r);
    return;
  }
  const uint32_t per_vec = 16 / elem, n = row_run<POW2>(r, nt) * per_vec;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
  for (uint32_t h = warp; h < nh; h += nwarps) {
    for (uint32_t e = lane; e < n; e += 32) {
      const uint32_t v = e / per_vec, within = (e - v * per_vec) * elem;
      const uint8_t* sp = sb + h * S.head_stride + row_offset<POW2>(r, v, S.tok_stride) + within;
      uint8_t* dp = db + h * D.head_stride + row_offset<POW2>(r, v, D.tok_stride) + within;
      if (elem == 2) *reinterpret_cast<uint16_t*>(dp) = *reinterpret_cast<const uint16_t*>(sp);
      else if (elem == 4) *reinterpret_cast<uint32_t*>(dp) = *reinterpret_cast<const uint32_t*>(sp);
      else *reinterpret_cast<uint2*>(dp) = *reinterpret_cast<const uint2*>(sp);
    }
  }
}

// The (layer l, outer o) region of a side of a paged transform, before any block offset.
__device__ __forceinline__ uint8_t* side_region(const PermuteSide& X, uint32_t l, uint32_t o)
{
  return reinterpret_cast<uint8_t*>(static_cast<uintptr_t>(__ldg(X.layer_base + (X.universal ? 0 : l)))) + l * X.layer_step +
         o * X.outer_step;
}

// The same region in block ids[i] of the side's table.  The sum is written out in this order rather than as side_region() plus
// the block offset: the other order costs the paged permute up to 15 more registers (53 -> 68 uncast).
__device__ __forceinline__ uint8_t* side_block(const PermuteSide& X, uint32_t i, uint32_t l, uint32_t o)
{
  return reinterpret_cast<uint8_t*>(static_cast<uintptr_t>(__ldg(X.layer_base + (X.universal ? 0 : l)))) +
         static_cast<uint64_t>(__ldg(X.ids + i)) * X.block_stride + l * X.layer_step + o * X.outer_step;
}

// Paged permute: the walk with the bases computed from the pools' layouts and block tables instead of host-built pointer
// tables, for any pair of KvBlockLayouts, optionally casting (CAST: KVBM_CAST_*; each side's strides are for its own row and
// its own head count).  nh heads of every unit move: source heads from s_win / head_stride on, destination heads from
// d_win / head_stride on (s_win, d_win: the head windows' byte offsets; 0 for every head of both sides).  One CTA per
// (block pair, layer, outer), also for a window of one head: packing several units of a narrow window into one CTA measured
// no faster (DESIGN §4.2b).  SCALED: the cast applies scales[l * no + o], loaded once per CTA.
template <int CAST, bool POW2, bool SCALED = false>
__global__ void __launch_bounds__(256)
kvbm_paged_permute_kernel(const __grid_constant__ PermuteSide S, const __grid_constant__ PermuteSide D, uint32_t layer_begin,
                          uint32_t nlayers, uint32_t no, uint32_t nh, uint32_t nt, RowSplit r, uint64_t s_win, uint64_t d_win,
                          const float* scales)
{
  const uint32_t unit = blockIdx.x;  // (pair * nlayers + l) * no + o
  const uint32_t pair = unit / (nlayers * no);
  const uint32_t rem = unit - pair * (nlayers * no);
  const uint32_t l = layer_begin + rem / no, o = rem % no;
  const ptx::Scale scale = ptx::make_scale(SCALED ? __ldg(scales + l * no + o) : 1.f);
  walk_head_rows<CAST, POW2, SCALED>(side_block(S, pair, l, o) + s_win, S.head_stride, S.tok_stride, side_block(D, pair, l, o) + d_win,
                                     D.head_stride, D.tok_stride, threadIdx.x >> 5, blockDim.x >> 5, nh, nt, r, scale);
}

// The gather: several sources, each with its own pool, format, head count, head window and layer window, into one destination.
// The covered destination heads are numbered 0 .. covered-1; entry[j] names the source of covered head j, which is head
// j - first of that source's window.  s_win / d_win: the window's first head on either side, in bytes.  A layer window maps
// source layers [src_begin, src_begin + count) to destination layers [dst_begin, dst_begin + count); sources with one
// destination window form a stage (DESIGN §4.2e).  Stage k covers destination layers [begin, end) and map entries first ..
// first + count - 1 (the map runs stage by stage, in source order within a stage), `sources` is the mask of its sources, and
// shift[s] is source s's layer minus the destination's.  The stages ascend and tile the launch's layer range: a gather without
// layer windows (a PP1 plan) is one stage over every layer, every shift 0.
struct GatherSource {
  PermuteSide S;
  uint64_t s_win, d_win;
  uint32_t first;
};
struct GatherStage {
  uint32_t begin, end, first, count, sources;
};
struct GatherParams {
  PermuteSide D;
  GatherSource src[KVBM_GATHER_MAX_SOURCES];
  uint8_t entry[KVBM_GATHER_MAX_HEADS];
  uint32_t covered;
  alignas(8) GatherStage stage[KVBM_GATHER_MAX_SOURCES];  // the measured layout: 4 B earlier reschedules the re-paging gathers
  uint32_t shift[KVBM_GATHER_MAX_SOURCES];
};

// The stage of destination layer l (one of the launch's range): the first stage that ends past it.  The scatter's params
// (ScatterParams) number their stages by source layer.
template <class Params>
__host__ __device__ __forceinline__ const GatherStage& stage_of(const Params& P, uint32_t l)
{
  uint32_t k = 0;
  while (l >= P.stage[k].end) ++k;
  return P.stage[k];
}

// One destination (block, layer, outer) unit of the gather, block `pair` of the tables, with one warp per covered destination
// head of layer l's stage T (looping by the CTA's warps past 8): every source's window of the unit is written by the same CTA, so
// a destination row that holds every head (OperationalNHD) is written whole by one CTA.  Each warp looks up its source and runs
// the same walk over one head, reading the source at its own layer l + shift.  SCALED: one scale array for every source,
// scales[l * no + o] by the destination layer, loaded once per unit.
template <int CAST, bool POW2, bool SCALED>
__device__ __forceinline__ void gather_unit(const GatherParams& P, const GatherStage& T, uint32_t pair, uint32_t l, uint32_t o, uint32_t no,
                                            uint32_t nt, const RowSplit& r, const float* scales)
{
  uint8_t* db = side_block(P.D, pair, l, o);
  const ptx::Scale scale = ptx::make_scale(SCALED ? __ldg(scales + l * no + o) : 1.f);
  const uint32_t end = T.first + T.count;
  for (uint32_t j = T.first + (threadIdx.x >> 5); j < end; j += blockDim.x >> 5) {
    const uint32_t s = P.entry[j];
    const GatherSource& G = P.src[s];
    const uint32_t h = j - G.first;  // head h of the window: walk heads h .. h of the window's bases
    walk_head_rows<CAST, POW2, SCALED>(side_block(G.S, pair, l + P.shift[s], o) + G.s_win, G.S.head_stride, G.S.tok_stride, db + G.d_win,
                                       P.D.head_stride, P.D.tok_stride, h, 1, h + 1, nt, r, scale);
  }
}

// One CTA per destination unit, as the paged permute.
template <int CAST, bool POW2, bool SCALED = false>
__global__ void __launch_bounds__(256)
kvbm_paged_gather_kernel(const __grid_constant__ GatherParams P, uint32_t layer_begin, uint32_t nlayers, uint32_t no, uint32_t nt, RowSplit r,
                         const float* scales)
{
  const uint32_t unit = blockIdx.x;  // (pair * nlayers + l) * no + o
  const uint32_t pair = unit / (nlayers * no);
  const uint32_t rem = unit - pair * (nlayers * no);
  const uint32_t l = layer_begin + rem / no;
  gather_unit<CAST, POW2, SCALED>(P, stage_of(P, l), pair, l, rem % no, no, nt, r, scales);
}

// Re-paging: a token range [token_begin, token_end) of one sequence between two block tables whose page sizes differ (one divides
// the other).  Sequence token p sits in slot p % P of block ids[p / P - first] on each side, P being that side's page.  `big` is
// the side with the larger page (the source on a tie), `small` the other; each side's strides are those of its own page.  One
// CTA per (big block, layer, outer) unit, clipped to the token range, one warp per head.  Within a head the lane's vector v is
// (token t of the unit, 16 B column c) by the row split; the token's slot in the big block is q = q0 + t, its small block and
// slot come from q by the page split (a shift and a mask, or a multiply-high exact for q < 2^32 / small_page).  The walk runs
// over all the unit's tokens, so one-token pages still keep 8 independent 16 B loads per lane in flight.
struct RepageGeom {
  RowSplit page;          // q -> (small block, slot): log2 / magic of the small page
  uint32_t small_page;
  uint32_t big_page;
  uint32_t ratio;         // big_page / small_page
  uint32_t big_first;     // token_begin / big_page: the big side's ids start at this block of the sequence
  uint32_t small_first;   // token_begin / small_page
  uint32_t token_begin, token_end;
  uint32_t layer_begin, nlayers, no, nh;
  uint32_t src_small;     // 1: the source is the small side
};
struct RepageParams {
  PermuteSide big, small;
  RepageGeom g;
};

// Big block j of the range (entry j of the big side's table), clipped to the token range: the slot q0 of its first token in
// the range, its token count, and small_k, the small table's entry of its first small block.  small_k wraps below 0 in the
// unit whose first small blocks lie before the range, and small_k + b (b >= those blocks) wraps back: index in uint32, never
// offset the pointer by it.
struct RepageUnit {
  uint32_t q0, tokens, small_k;
};
__device__ __forceinline__ RepageUnit repage_unit(const RepageGeom& G, uint32_t j)
{
  const uint32_t first = (G.big_first + j) * G.big_page;  // sequence position of the big block's slot 0
  const uint32_t t0 = max(G.token_begin, first), t1 = min(G.token_end, first + G.big_page);
  return {t0 - first, t1 - t0, (G.big_first + j) * G.ratio - G.small_first};
}

// Where a re-paging launch's units come from.  kRange: the launch's one token range (repage_unit).  Every other kind is a batch
// of sequences whose unit j is record j of a 16 B unit table: the same three words, whose small_k indexes the concatenated small
// table, in one 16 B load where a search over per-sequence prefix sums would be log2(n) dependent loads at the head of a CTA that
// lives a few microseconds.  The kinds differ in what the record's fourth word means:
//   kSeqs         kvbm_repage_unit           the sequence index (unused by the walks)
//   kRouted       kvbm_route_unit            the sequence's rank mask (a scatter's targets, a gather's sources)
//   kPhased       kvbm_repage_anypage_unit   the phase, for pages that need not divide (DESIGN §4.2k)
//   kRoutedPhased kvbm_route_anypage_unit    mask | phase << 16 (DESIGN §4.2m)
enum RepageUnits { kRange, kSeqs, kRouted, kPhased, kRoutedPhased };
__host__ __device__ constexpr bool routed_units(RepageUnits k) { return k == kRouted || k == kRoutedPhased; }
__host__ __device__ constexpr bool phased_units(RepageUnits k) { return k == kPhased || k == kRoutedPhased; }

// Unit j of a re-paging launch whose units are UNITS, with its rank mask and its phase (the slot of small block small_k that
// holds the big block's slot 0), each 0 where the kind has none.  table: the unit table (unused for kRange).
struct RepageUnitRecord {
  RepageUnit u;
  uint32_t mask, phase;
};
template <RepageUnits UNITS>
__device__ __forceinline__ RepageUnitRecord load_unit(const RepageGeom& G, const void* table, uint32_t j)
{
  if constexpr (UNITS == kRange) {
    return {repage_unit(G, j), 0, 0};
  } else {
    const uint4 w = __ldg(static_cast<const uint4*>(table) + j);
    if constexpr (UNITS == kSeqs) return {{w.x, w.y, w.z}, 0, 0};
    if constexpr (UNITS == kRouted) return {{w.x, w.y, w.z}, w.w, 0};
    if constexpr (UNITS == kPhased) return {{w.x, w.y, w.z}, 0, w.w};
    // kRoutedPhased: the mask is cut to its 16 bits although the walks only read bits below the launch's rank count, so that the
    // phase never reaches a mask reader.
    return {{w.x, w.y, w.z}, w.w & 0xFFFFu, w.w >> 16};
  }
}

// The unit of a one-CTA-per-unit re-paging kernel, blockIdx.x = (big block j * nlayers + l - layer_begin) * no + o.  The caller
// takes o = rem % no itself: the gathers after their stage lookup, the scatters before it.  Moving it changes how ptxas
// schedules the division.
struct RepageCta {
  uint32_t j, l, rem;
};
__device__ __forceinline__ RepageCta repage_cta(const RepageGeom& G)
{
  const uint32_t unit = blockIdx.x;
  const uint32_t j = unit / (G.nlayers * G.no);
  const uint32_t rem = unit - j * (G.nlayers * G.no);
  return {j, G.layer_begin + rem / G.no, rem};
}

// Where 16 B vector vv of a re-paging head's run sits: its 16 B column c, its token's slot q in the big block, and the small
// block (entry small_k + b of the small table) and slot that hold the same token.  PHASE: pages that need not divide (DESIGN
// §4.2k), where the big block's slot 0 sits at slot `phase` of small block small_k, so the small side splits phase + q; the big
// side's address still takes q.  phase + q < big_page + small_page - gcd, which keeps the multiply-high exact under
// repage_pages' bound.  Without PHASE the small side splits q itself.
struct RepageAt {
  uint32_t c, q, b, slot;
};
template <bool POW2, bool PPOW2, bool PHASE = false>
__device__ __forceinline__ RepageAt repage_at(const RepageGeom& G, const RowSplit& r, uint32_t q0, uint32_t vv, uint32_t phase = 0)
{
  const uint32_t t = POW2 ? vv >> r.vpr : __umulhi(vv, r.magic);
  const uint32_t c = POW2 ? vv & ((1u << r.vpr) - 1) : vv - t * r.vpr;
  const uint32_t q = q0 + t;
  const uint32_t qs = PHASE ? phase + q : q;
  const uint32_t b = PPOW2 ? qs >> G.page.vpr : __umulhi(qs, G.page.magic);
  const uint32_t slot = PPOW2 ? qs & (G.small_page - 1) : qs - b * G.small_page;
  return {c, q, b, slot};
}

// The vector's address on the big side (bh: the head's rows in the big block) and on the small side (sh: the head's rows in the
// small side's (layer, outer) region, before the block offset; small block b is entry small_k + b of small_ids, RepageUnit).
__device__ __forceinline__ const uint8_t* repage_big(const uint8_t* bh, uint32_t big_tok, uint32_t big_shift, const RepageAt& a)
{
  return bh + a.q * big_tok + (a.c << big_shift);
}
__device__ __forceinline__ const uint8_t* repage_small(const uint8_t* sh, const int32_t* small_ids, uint32_t small_k,
                                                       uint64_t small_block_stride, uint32_t small_tok, uint32_t small_shift, const RepageAt& a)
{
  return sh + static_cast<uint64_t>(__ldg(small_ids + (small_k + a.b))) * small_block_stride + a.slot * small_tok + (a.c << small_shift);
}

// The load half of a re-paging walk: the IN 16 B loads of one vector.  The store half: the OUT 16 B stores of one vector as the
// destination holds it -- the loaded vector itself without a cast, else cast_vector's result (bit for bit the paged permute's
// cast), which a scatter computes once and stores to every destination of the vector.
template <int IN>
__device__ __forceinline__ void load_vector(const uint8_t* s, uint4 (&x)[IN])
{
#pragma unroll
  for (int i = 0; i < IN; ++i) x[i] = ptx::ld_stream_v4(s + 16 * i);
}
template <int OUT>
__device__ __forceinline__ void store_vector(const uint8_t* d, const uint4 (&y)[OUT])
{
#pragma unroll
  for (int i = 0; i < OUT; ++i) ptx::st_stream_v4(const_cast<uint8_t*>(d) + 16 * i, y[i]);
}

// One head of a re-paging unit: its run of `run` 16 B vectors from slot q0 of the big block on.  bh: the head's rows in the
// big block; sh: its rows in the small side's (layer, outer) region, before the block offset.  Small block b of the unit is
// entry small_k + b of small_ids (RepageUnit).  Every re-paging kernel but the scatter runs its heads through this loop.  PHASE /
// phase: repage_at's, the unit's phase when pages need not divide.
template <int CAST, bool POW2, bool SCALED, bool PPOW2, bool PHASE = false>
__device__ __forceinline__ void repage_head_rows(const uint8_t* bh, uint32_t big_tok, uint32_t big_shift, const uint8_t* sh,
                                                 const int32_t* small_ids, uint32_t small_k, uint64_t small_block_stride,
                                                 uint32_t small_tok, uint32_t small_shift, const RepageGeom& G, uint32_t q0,
                                                 uint32_t run, const RowSplit& r, const ptx::Scale& scale, uint32_t phase = 0)
{
  constexpr int IN = CAST == KVBM_CAST_BF16_TO_FP8E4M3 ? 2 : 1;   // 16 B loads per vector
  constexpr int OUT = CAST == KVBM_CAST_FP8E4M3_TO_BF16 ? 2 : 1;  // 16 B stores per vector
  constexpr int U = 8 / IN;
  const int lane = threadIdx.x & 31;
  for (uint32_t v = lane; v < run; v += U * 32) {
    uint4 x[U][IN];
    uint8_t* dp[U];
#pragma unroll
    for (int k = 0; k < U; ++k)
      if (v + k * 32 < run) {
        const RepageAt a = repage_at<POW2, PPOW2, PHASE>(G, r, q0, v + k * 32, phase);
        const uint8_t* big_p = repage_big(bh, big_tok, big_shift, a);
        const uint8_t* small_p = repage_small(sh, small_ids, small_k, small_block_stride, small_tok, small_shift, a);
        const uint8_t* s = G.src_small ? small_p : big_p;
        dp[k] = const_cast<uint8_t*>(G.src_small ? big_p : small_p);
        load_vector(s, x[k]);
      }
#pragma unroll
    for (int k = 0; k < U; ++k)
      if (v + k * 32 < run) {
        if constexpr (CAST == KVBM_CAST_NONE) {
          store_vector(dp[k], x[k]);
        } else {
          uint4 y[OUT];
          cast_vector<SCALED>(x[k], y, scale);
          store_vector(dp[k], y);
        }
      }
  }
}

template <int CAST, bool POW2, bool SCALED, bool PPOW2>
__global__ void __launch_bounds__(256)
kvbm_paged_repage_kernel(const __grid_constant__ RepageParams P, RowSplit r, const float* scales)
{
  constexpr int IN = CAST == KVBM_CAST_BF16_TO_FP8E4M3 ? 2 : 1;
  constexpr int OUT = CAST == KVBM_CAST_FP8E4M3_TO_BF16 ? 2 : 1;
  const auto [j, l, rem] = repage_cta(P.g);
  const uint32_t o = rem % P.g.no;
  const RepageUnit u = repage_unit(P.g, j);
  const uint8_t* big_base = side_block(P.big, j, l, o);
  const uint8_t* small_base = side_region(P.small, l, o);
  const ptx::Scale scale = ptx::make_scale(SCALED ? __ldg(scales + l * P.g.no + o) : 1.f);
  // column shifts of either side: the source's vector is 16 * IN bytes, the destination's 16 * OUT
  const uint32_t big_shift = P.g.src_small ? 3 + OUT : 3 + IN, small_shift = P.g.src_small ? 3 + IN : 3 + OUT;
  const uint32_t run = row_run<POW2>(r, u.tokens);
  for (uint32_t h = threadIdx.x >> 5; h < P.g.nh; h += blockDim.x >> 5)
    repage_head_rows<CAST, POW2, SCALED, PPOW2>(big_base + h * P.big.head_stride, static_cast<uint32_t>(P.big.tok_stride), big_shift,
                                                small_base + h * P.small.head_stride, P.small.ids, u.small_k, P.small.block_stride,
                                                static_cast<uint32_t>(P.small.tok_stride), small_shift, P.g, u.q0, run, r, scale);
}

// Re-paging and the gather in one launch: several sources with one page size Ps (a prefill TP or PP x TP group), each with its
// own pool, format, head count, head window and layer window, into one destination of page Pd, over a token range.  The unit is
// the re-paging one: one CTA per (block of the larger-page side, layer, outer), clipped to the range; the warps are the
// gather's: one per covered destination head of the layer's stage, looping by the CTA's warps past 8, each finding its source
// through the head map and reading it at its own layer.  All sources share Ps and the range, so big block j names the same
// sequence positions in every source: when the sources have the larger page each warp reads block j of its own table; when the
// destination has it, a unit is one destination block and one CTA writes whole rows of an OperationalNHD destination.  The
// small side's block comes per 16 B vector from the warp's own source table or the destination's.  geo.nh: the covered heads.
struct RepageGatherParams {
  GatherParams g;
  RepageGeom geo;
};

// Unit (big block j, destination layer l, outer o) of the re-paging gather: the warp of map entry k of l's stage T reads its source
// s at the source's own layer l + shift[s].  SCALED: one scale array for every source, scales[l * no + o] by the destination layer.
// UNITS / table: where the unit comes from (load_unit).  A routed kind walks only the entries of the stage's sources in the
// unit's mask, numbered densely (route_entry), so no warp idles on an unrouted window; heads[s] is source s's entry count.  Only
// the stage's sources are consulted, so mask bits at or above the launch's sources never are.  A phased kind's walks split the
// unit's phase (repage_head_rows' PHASE).
template <int CAST, bool POW2, bool SCALED, bool PPOW2, RepageUnits UNITS = kRange>
__device__ __forceinline__ void repage_gather_unit(const RepageGatherParams& P, const GatherStage& T, uint32_t j, uint32_t l, uint32_t o,
                                                   const RowSplit& r, const float* scales, const void* table = nullptr,
                                                   const uint16_t* heads = nullptr)
{
  constexpr int IN = CAST == KVBM_CAST_BF16_TO_FP8E4M3 ? 2 : 1;
  constexpr int OUT = CAST == KVBM_CAST_FP8E4M3_TO_BF16 ? 2 : 1;
  const GatherParams& g = P.g;
  const RepageGeom& G = P.geo;
  const uint32_t first = T.first, end = T.first + T.count;
  const PermuteSide& D = g.D;
  const RepageUnitRecord rec = load_unit<UNITS>(G, table, j);
  const RepageUnit u = rec.u;  // named, not bound: the walk's lambda captures them
  const uint32_t mask = rec.mask, phase = rec.phase;
  const uint8_t* d_region = side_region(D, l, o);
  const ptx::Scale scale = ptx::make_scale(SCALED ? __ldg(scales + l * G.no + o) : 1.f);
  const uint32_t big_shift = G.src_small ? 3 + OUT : 3 + IN, small_shift = G.src_small ? 3 + IN : 3 + OUT;
  const uint32_t run = row_run<POW2>(r, u.tokens);
  // map entry k of source s (head h = k - first of its window)
  auto head = [&](uint32_t k, uint32_t s) {
    const GatherSource& S = g.src[s];
    const uint32_t h = k - S.first;  // head h of the window
    const uint8_t* sh = side_region(S.S, l + g.shift[s], o) + S.s_win + h * S.S.head_stride;
    const uint8_t* dh = d_region + S.d_win + h * D.head_stride;
    const bool ss = G.src_small;
    const PermuteSide& B = ss ? D : S.S;
    const PermuteSide& Sm = ss ? S.S : D;
    const uint8_t* bh = (ss ? dh : sh) + static_cast<uint64_t>(__ldg(B.ids + j)) * B.block_stride;
    repage_head_rows<CAST, POW2, SCALED, PPOW2, phased_units(UNITS)>(bh, static_cast<uint32_t>(B.tok_stride), big_shift, ss ? sh : dh, Sm.ids,
                                                                     u.small_k, Sm.block_stride, static_cast<uint32_t>(Sm.tok_stride),
                                                                     small_shift, G, u.q0, run, r, scale, phase);
  };
  if constexpr (routed_units(UNITS)) {
    // routed entry i of the unit: the stage's map runs source by source in source order, so skip whole sources up to it
    const uint32_t warps = blockDim.x >> 5;
    uint32_t i = threadIdx.x >> 5;
    for (uint32_t rest = T.sources & mask; rest != 0; rest &= rest - 1) {
      const uint32_t s = __ffs(rest) - 1, n = heads[s], at = g.src[s].first;
      for (; i < n; i += warps) head(at + i, s);
      i -= n;
    }
  } else {
    for (uint32_t k = first + (threadIdx.x >> 5); k < end; k += blockDim.x >> 5) head(k, g.entry[k]);
  }
}

// Three CTAs per SM (at most 80 registers): the stage lookup otherwise takes the scaled fp8 -> bf16 walk with a power-of-two
// row and page to 86 registers, and to two CTAs per SM.
template <int CAST, bool POW2, bool SCALED, bool PPOW2>
__global__ void __launch_bounds__(256, 3)
kvbm_paged_repage_gather_kernel(const __grid_constant__ RepageGatherParams P, RowSplit r, const float* scales)
{
  const auto [j, l, rem] = repage_cta(P.geo);
  repage_gather_unit<CAST, POW2, SCALED, PPOW2>(P, stage_of(P.g, l), j, l, rem % P.geo.no, r, scales);
}

// kvbm_paged_repage_gather_kernel over a batch of sequences: big block j is entry j of the concatenated big table and record j
// of `units`; geo's token range and first blocks are unused.  The same bound: three CTAs per SM.
template <int CAST, bool POW2, bool SCALED, bool PPOW2>
__global__ void __launch_bounds__(256, 3)
kvbm_paged_batch_repage_gather_kernel(const __grid_constant__ RepageGatherParams P, const kvbm_repage_unit* units, RowSplit r, const float* scales)
{
  const auto [j, l, rem] = repage_cta(P.geo);
  repage_gather_unit<CAST, POW2, SCALED, PPOW2, kSeqs>(P, stage_of(P.g, l), j, l, rem % P.geo.no, r, scales, units);
}

// Each source's entry count in the head map (its window's heads), which a routed unit needs to skip unrouted sources.
struct SourceHeads {
  uint16_t n[KVBM_GATHER_MAX_SOURCES];
};

// kvbm_paged_batch_repage_gather_kernel over a routed batch: record j of `routes` also names the sources big block j reads, and
// only their entries are walked.  The same bound: three CTAs per SM.
template <int CAST, bool POW2, bool SCALED, bool PPOW2>
__global__ void __launch_bounds__(256, 3)
kvbm_paged_repage_fanin_kernel(const __grid_constant__ RepageGatherParams P, const __grid_constant__ SourceHeads H, const kvbm_route_unit* routes,
                               RowSplit r, const float* scales)
{
  const auto [j, l, rem] = repage_cta(P.geo);
  repage_gather_unit<CAST, POW2, SCALED, PPOW2, kRouted>(P, stage_of(P.g, l), j, l, rem % P.geo.no, r, scales, routes, H.n);
}

// kvbm_paged_batch_repage_gather_kernel over a batch whose pages need not divide: record j of `units` also carries big block j's
// phase (DESIGN §4.2k).  The same bound: three CTAs per SM.
template <int CAST, bool POW2, bool SCALED, bool PPOW2>
__global__ void __launch_bounds__(256, 3)
kvbm_paged_repage_anypage_kernel(const __grid_constant__ RepageGatherParams P, const kvbm_repage_anypage_unit* units, RowSplit r,
                                 const float* scales)
{
  const auto [j, l, rem] = repage_cta(P.geo);
  repage_gather_unit<CAST, POW2, SCALED, PPOW2, kPhased>(P, stage_of(P.g, l), j, l, rem % P.geo.no, r, scales, units);
}

// kvbm_paged_repage_fanin_kernel over a batch whose pages need not divide: record j of `units` carries big block j's sources and
// phase in its fourth word (DESIGN §4.2m).  The same bound: three CTAs per SM.
template <int CAST, bool POW2, bool SCALED, bool PPOW2>
__global__ void __launch_bounds__(256, 3)
kvbm_paged_repage_collect_kernel(const __grid_constant__ RepageGatherParams P, const __grid_constant__ SourceHeads H,
                                 const kvbm_route_anypage_unit* units, RowSplit r, const float* scales)
{
  const auto [j, l, rem] = repage_cta(P.geo);
  repage_gather_unit<CAST, POW2, SCALED, PPOW2, kRoutedPhased>(P, stage_of(P.g, l), j, l, rem % P.geo.no, r, scales, units, H.n);
}

// The re-paging scatter, the gather's mirror image: ONE source pool of page Ps (a prefill rank) into up to
// KVBM_GATHER_MAX_SOURCES targets of page Pd, each a destination pool's side with its own format, table and head count, one head
// window and one layer window; a pool may appear in several targets.  Targets with one source layer window form a stage; the
// stages ascend in source layers and tile the launch's (source) layer range.  The covered source heads of every stage are numbered
// entry 0 .. entries-1, stage by stage in ascending head order: head[k] is entry k's source head, and pairs pair_first[k] ..
// pair_first[k + 1] - 1 its (target, destination head) pairs, pair_tgt[p] naming the target, whose destination head is the source
// head plus head_delta and whose destination layer the source layer plus shift (both modulo 2^32).
struct ScatterTarget {
  PermuteSide D;
  uint32_t shift, head_delta;
};
struct ScatterParams {
  PermuteSide S;
  ScatterTarget tgt[KVBM_GATHER_MAX_SOURCES];
  RepageGeom geo;
  GatherStage stage[KVBM_GATHER_MAX_SOURCES];  // begin / end: source layers; first / count: entries
  uint32_t head[KVBM_GATHER_MAX_HEADS];
  uint16_t pair_first[KVBM_GATHER_MAX_HEADS + 1];
  uint8_t pair_tgt[KVBM_GATHER_MAX_HEADS];
};

// The layer of source s that a unit of launch layer l reads: a gather's source at its own shift, the scatter's one source at l.
__host__ __device__ __forceinline__ uint32_t source_layer(const GatherParams& P, int s, uint32_t l) { return l + P.shift[s]; }
__host__ __device__ __forceinline__ uint32_t source_layer(const ScatterParams&, int, uint32_t l) { return l; }

// One covered source head (entry k) of a scatter unit (big block j, source layer l, outer o): the re-paging walk's load half reads
// each 16 B vector ONCE and casts it once, and its store half writes it to every (target, destination head) pair of the entry,
// each at its own layer.  With Ps >= Pd block j is the source's and each target finds the vector's small block in its own table;
// with Ps < Pd block j is entry j of every target's table (they share Pd and the range).
// ROUTE: only the pairs whose target's bit is set in `mask` (the unit's sequence's targets) are stored, and an entry with no such
// pair loads nothing.  Only pair_tgt[p] < num_targets selects a bit, so bits at or above the launch's target count are never read.
// PHASE / phase: repage_at's, the unit's phase when pages need not divide (DESIGN §4.2l).  Both halves split phase + q on the small
// side: with Ps < Pd the loads from the source's table, else every target's stores into its own table, all with the one small_k
// and phase (every target shares Pd and the batch layout).
template <int CAST, bool POW2, bool SCALED, bool PPOW2, bool ROUTE = false, bool PHASE = false>
__device__ __forceinline__ void scatter_head_rows(const ScatterParams& P, uint32_t k, uint32_t j, uint32_t l, uint32_t o, const RepageUnit& u,
                                                  uint32_t run, const RowSplit& r, const ptx::Scale& scale, uint32_t mask = 0,
                                                  uint32_t phase = 0)
{
  constexpr int IN = CAST == KVBM_CAST_BF16_TO_FP8E4M3 ? 2 : 1;
  constexpr int OUT = CAST == KVBM_CAST_FP8E4M3_TO_BF16 ? 2 : 1;
  constexpr int U = 8 / IN;
  const RepageGeom& G = P.geo;
  const PermuteSide& S = P.S;
  const bool ss = G.src_small;
  const uint32_t big_shift = ss ? 3 + OUT : 3 + IN, small_shift = ss ? 3 + IN : 3 + OUT;
  const uint32_t h = P.head[k], p0 = P.pair_first[k], p1 = P.pair_first[k + 1];
  if constexpr (ROUTE) {
    uint32_t routed = 0;
    for (uint32_t p = p0; p < p1; ++p) routed |= (mask >> P.pair_tgt[p]) & 1u;
    if (!routed) return;
  }
  const uint8_t* sh = (ss ? side_region(S, l, o) : side_block(S, j, l, o)) + h * S.head_stride;
  const int lane = threadIdx.x & 31;
  for (uint32_t v = lane; v < run; v += U * 32) {
    uint4 x[U][IN];
#pragma unroll
    for (int i = 0; i < U; ++i)
      if (v + i * 32 < run) {
        const RepageAt a = repage_at<POW2, PPOW2, PHASE>(G, r, u.q0, v + i * 32, phase);
        load_vector(ss ? repage_small(sh, S.ids, u.small_k, S.block_stride, static_cast<uint32_t>(S.tok_stride), small_shift, a)
                       : repage_big(sh, static_cast<uint32_t>(S.tok_stride), big_shift, a),
                    x[i]);
      }
#pragma unroll
    for (int i = 0; i < U; ++i)
      if (v + i * 32 < run) {
        const RepageAt a = repage_at<POW2, PPOW2, PHASE>(G, r, u.q0, v + i * 32, phase);
        uint4 y[OUT];
        if constexpr (CAST == KVBM_CAST_NONE)
          y[0] = x[i][0];
        else
          cast_vector<SCALED>(x[i], y, scale);
#pragma unroll 1
        for (uint32_t p = p0; p < p1; ++p) {
          if constexpr (ROUTE)
            if (!((mask >> P.pair_tgt[p]) & 1u)) continue;
          const ScatterTarget& T = P.tgt[P.pair_tgt[p]];
          const PermuteSide& D = T.D;
          const uint32_t dl = l + T.shift;
          const uint8_t* dh = (ss ? side_block(D, j, dl, o) : side_region(D, dl, o)) + (h + T.head_delta) * D.head_stride;
          store_vector(ss ? repage_big(dh, static_cast<uint32_t>(D.tok_stride), big_shift, a)
                          : repage_small(dh, D.ids, u.small_k, D.block_stride, static_cast<uint32_t>(D.tok_stride), small_shift, a),
                       y);
        }
      }
  }
}

// One (big block j, source layer l, outer o) unit of the scatter, clipped to the range, with l's stage T: one warp per covered
// source head of T, looping by the CTA's warps past 8.  SCALED: the SOURCE's scales[l * no + o], loaded once per unit.
// UNITS / table: where the unit comes from (load_unit); a routed kind's mask and a phased kind's phase go to scatter_head_rows.
template <int CAST, bool POW2, bool SCALED, bool PPOW2, RepageUnits UNITS = kRange>
__device__ __forceinline__ void scatter_unit(const ScatterParams& P, const GatherStage& T, uint32_t j, uint32_t l, uint32_t o, const RowSplit& r,
                                             const float* scales, const void* table = nullptr)
{
  const RepageGeom& G = P.geo;
  const RepageUnitRecord rec = load_unit<UNITS>(G, table, j);
  const ptx::Scale scale = ptx::make_scale(SCALED ? __ldg(scales + l * G.no + o) : 1.f);
  const uint32_t run = row_run<POW2>(r, rec.u.tokens);
  const uint32_t end = T.first + T.count;
  for (uint32_t k = T.first + (threadIdx.x >> 5); k < end; k += blockDim.x >> 5)
    scatter_head_rows<CAST, POW2, SCALED, PPOW2, routed_units(UNITS), phased_units(UNITS)>(P, k, j, l, o, rec.u, run, r, scale, rec.mask,
                                                                                           rec.phase);
}

// One CTA per unit, as the re-paging gather.  The re-paging gathers' bound: three CTAs per SM.
template <int CAST, bool POW2, bool SCALED, bool PPOW2>
__global__ void __launch_bounds__(256, 3)
kvbm_paged_repage_scatter_kernel(const __grid_constant__ ScatterParams P, RowSplit r, const float* scales)
{
  const auto [j, l, rem] = repage_cta(P.geo);
  const uint32_t o = rem % P.geo.no;
  scatter_unit<CAST, POW2, SCALED, PPOW2>(P, stage_of(P, l), j, l, o, r, scales);
}

// kvbm_paged_repage_scatter_kernel over a batch of sequences: big block j is entry j of the concatenated big table (the source's,
// or every target's: they share Pd and the batch) and record j of `units`; geo's token range and first blocks are unused.  The
// same bound: three CTAs per SM.
template <int CAST, bool POW2, bool SCALED, bool PPOW2>
__global__ void __launch_bounds__(256, 3)
kvbm_paged_repage_push_seqs_kernel(const __grid_constant__ ScatterParams P, const kvbm_repage_unit* units, RowSplit r, const float* scales)
{
  const auto [j, l, rem] = repage_cta(P.geo);
  const uint32_t o = rem % P.geo.no;
  scatter_unit<CAST, POW2, SCALED, PPOW2, kSeqs>(P, stage_of(P, l), j, l, o, r, scales, units);
}

// kvbm_paged_repage_push_seqs_kernel over a routed batch: record j of `routes` also names the targets big block j goes to, and
// only those are written.  The same bound: three CTAs per SM.
template <int CAST, bool POW2, bool SCALED, bool PPOW2>
__global__ void __launch_bounds__(256, 3)
kvbm_paged_repage_route_kernel(const __grid_constant__ ScatterParams P, const kvbm_route_unit* routes, RowSplit r, const float* scales)
{
  const auto [j, l, rem] = repage_cta(P.geo);
  const uint32_t o = rem % P.geo.no;
  scatter_unit<CAST, POW2, SCALED, PPOW2, kRouted>(P, stage_of(P, l), j, l, o, r, scales, routes);
}

// kvbm_paged_repage_push_seqs_kernel over a batch whose pages need not divide: record j of `units` also carries big block j's phase
// (DESIGN §4.2l).  The same bound: three CTAs per SM.
template <int CAST, bool POW2, bool SCALED, bool PPOW2>
__global__ void __launch_bounds__(256, 3)
kvbm_paged_repage_phased_push_kernel(const __grid_constant__ ScatterParams P, const kvbm_repage_anypage_unit* units, RowSplit r,
                                     const float* scales)
{
  const auto [j, l, rem] = repage_cta(P.geo);
  const uint32_t o = rem % P.geo.no;
  scatter_unit<CAST, POW2, SCALED, PPOW2, kPhased>(P, stage_of(P, l), j, l, o, r, scales, units);
}

// kvbm_paged_repage_route_kernel over a batch whose pages need not divide: record j of `units` carries big block j's targets and
// phase in its fourth word (DESIGN §4.2m).  The same bound: three CTAs per SM.
template <int CAST, bool POW2, bool SCALED, bool PPOW2>
__global__ void __launch_bounds__(256, 3)
kvbm_paged_repage_deal_kernel(const __grid_constant__ ScatterParams P, const kvbm_route_anypage_unit* units, RowSplit r, const float* scales)
{
  const auto [j, l, rem] = repage_cta(P.geo);
  const uint32_t o = rem % P.geo.no;
  scatter_unit<CAST, POW2, SCALED, PPOW2, kRoutedPhased>(P, stage_of(P, l), j, l, o, r, scales, units);
}

// The scatter's signal after its launch: every target's done flag (epoch) and the completion word, system scope.
struct ScatterFlags {
  uint32_t* done[KVBM_GATHER_MAX_SOURCES];
};
__global__ void kvbm_scatter_signal_kernel(const ScatterFlags F, int n, uint32_t epoch, uint32_t* completion, uint32_t completion_value)
{
  __threadfence_system();
  for (int t = 0; t < n; ++t)
    if (F.done[t]) ptx::st_release_sys(F.done[t], epoch);
  if (completion) ptx::st_release_sys(completion, completion_value);
}

// ------------------------------------------------------------------------------------------------
// Layer streaming of the permuting and re-paging gathers (kvbm_permute_stream, spinning form).  The ungated kernels are one
// CTA per unit in block-major order, scheduled by the hardware: gating them would fill the GPU with spinners that starve the
// producer.  The gated kernels are a persistent grid instead: each CTA claims a batch of `batch` consecutive units per ticket
// from the ticket word ctl[2] in LAYER-major order, waits once per layer it enters for the flags of that layer's stage (warp
// 0, wait_layer_ready's relaxed polls, acquire fence, timeout and abort word), walks each unit with the ungated kernel's
// unit body (gather_unit / repage_gather_unit), and publishes what it moved of a layer -- every thread fences its stores, one barrier, one arrive_layer with
// the count -- when the batch ends and before it enters another layer.  So a CTA publishes every unit before it can wait on a
// later layer: a receiver that releases layer l + 1 only after seeing layer l done cannot dead-lock against it, and a batch that
// crosses a stage boundary gates on the next stage's sources when it enters that layer.  The warps of a CTA run on into the
// batch's next unit without waiting for each other.  The last CTA to finish runs arrive_transfer (re-zeroes the workspace, done
// / completion flags, or 0xFFFFFFFF on abort).
// ------------------------------------------------------------------------------------------------
struct GateArgs {
  StreamSync ss;  // ndst 1: the destination's layer_done / done flags; items = units; total_rings = CTAs
  const uint32_t* ready[KVBM_GATHER_MAX_SOURCES];
  int num_ready;
};

// The ready flags of the sources of layer l's stage T, each at its own layer (source_layer), waited for by warp 0; the verdict
// goes to the whole CTA.  False: the transfer aborted.
template <class Params>
__device__ __forceinline__ bool gate_layer(const GateArgs& A, const Params& P, const GatherStage& T, uint32_t l, uint32_t* s_ok)
{
  if (threadIdx.x < 32) {
    bool ok = true;
    for (int s = 0; s < A.num_ready && ok; ++s)
      if ((T.sources >> s) & 1u) {
        StreamSync w = A.ss;
        w.layer_ready = A.ready[s];
        ok = wait_layer_ready(w, static_cast<int>(source_layer(P, s, l)), threadIdx.x);
      }
    if (threadIdx.x == 0) *s_ok = ok ? 1u : 0u;
  }
  __syncthreads();
  return *s_ok != 0;
}

// `count` units of layer l are done: their stores are visible at gpu scope before thread 0 counts them (arrive_layer's acq_rel
// atomic; the CTA that completes a layer adds the system-scope fence before the flag).  The barrier also ends every thread's
// reads of the shared claim word.
__device__ __forceinline__ void publish_units(const GateArgs& A, uint32_t l, uint32_t count)
{
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0 && A.ss.want_layers && count != 0) arrive_layer(A.ss, static_cast<int>(l), count);
}

// The claim / gate / publish loop of every gated kernel over units [0, total) of the gather or scatter P: layer_of(u) is unit u's
// absolute layer, walk(u, l, T) moves it with T its layer's stage, looked up once per layer the CTA enters.  more_done: the
// last CTA's done flags besides A.ss's own (arrive_transfer).
template <class Params, class LayerOf, class Walk, class MoreDone = NoMoreFlags>
__device__ __forceinline__ void gated_units(const GateArgs& A, const Params& P, uint32_t total, uint32_t batch, LayerOf layer_of, Walk walk,
                                            MoreDone more_done = MoreDone{})
{
  __shared__ uint32_t s_ticket, s_ok;
  uint32_t entered = UINT32_MAX;
  GatherStage T{};
  for (;;) {
    if (threadIdx.x == 0) s_ticket = atomicAdd(A.ss.ctl + 2, 1u);
    __syncthreads();
    const uint64_t first = static_cast<uint64_t>(s_ticket) * batch;
    if (first >= total) break;
    const uint32_t last = static_cast<uint32_t>(min(first + batch, static_cast<uint64_t>(total)));
    uint32_t pending = 0;
    bool aborted = false;
    for (uint32_t u = static_cast<uint32_t>(first); u < last; ++u) {
      const uint32_t l = layer_of(u);
      if (l != entered) {
        if (pending != 0) publish_units(A, entered, pending);
        pending = 0;
        T = stage_of(P, l);
        if (!gate_layer(A, P, T, l, &s_ok)) {
          aborted = true;
          break;
        }
        entered = l;
      }
      walk(u, l, T);
      ++pending;
    }
    if (aborted) break;
    publish_units(A, entered, pending);
  }
  if (threadIdx.x == 0) arrive_transfer(A.ss, more_done);
}

// kvbm_paged_gather_kernel's unit walk behind the gate; unit = (l * num_blocks + pair) * no + o over the layer range.
template <int CAST, bool POW2, bool SCALED>
__global__ void __launch_bounds__(256, 1)
kvbm_gated_gather_kernel(const __grid_constant__ GatherParams P, const __grid_constant__ GateArgs A, uint32_t num_blocks, uint32_t layer_begin,
                         uint32_t nlayers, uint32_t no, uint32_t nt, RowSplit r, const float* scales, uint32_t batch)
{
  const uint32_t per_layer = num_blocks * no;
  gated_units(A, P, per_layer * nlayers, batch, [&](uint32_t u) { return layer_begin + u / per_layer; }, [&](uint32_t u, uint32_t l, const GatherStage& T) {
    const uint32_t rem = u - (l - layer_begin) * per_layer;
    const uint32_t pair = rem / no;
    gather_unit<CAST, POW2, SCALED>(P, T, pair, l, rem - pair * no, no, nt, r, scales);
  });
}

// gated_units over the units (l * num_big + j) * no + o of a re-paging launch's layer range G: unit(T, j, l, o) moves unit (big
// block j, layer l, outer o), T being l's stage in P.
template <class Params, class Unit, class MoreDone = NoMoreFlags>
__device__ __forceinline__ void gated_repage_units(const GateArgs& A, const Params& P, const RepageGeom& G, uint32_t num_big, uint32_t batch,
                                                   Unit unit, MoreDone more_done = MoreDone{})
{
  const uint32_t per_layer = num_big * G.no;
  gated_units(
      A, P, per_layer * G.nlayers, batch, [&](uint32_t u) { return G.layer_begin + u / per_layer; },
      [&, unit](uint32_t u, uint32_t l, const GatherStage& T) {  // `unit` by value: by reference, ptxas schedules the loop differently
        const uint32_t rem = u - (l - G.layer_begin) * per_layer;
        const uint32_t j = rem / G.no;
        unit(T, j, l, rem - j * G.no);
      },
      more_done);
}

// kvbm_paged_repage_gather_kernel's unit walk behind the gate; unit = (l * num_big + j) * no + o over the layer range.
template <int CAST, bool POW2, bool SCALED, bool PPOW2>
__global__ void __launch_bounds__(256)
kvbm_gated_repage_gather_kernel(const __grid_constant__ RepageGatherParams P, const __grid_constant__ GateArgs A, uint32_t num_big, RowSplit r,
                                const float* scales, uint32_t batch)
{
  gated_repage_units(A, P.g, P.geo, num_big, batch, [&](const GatherStage& T, uint32_t j, uint32_t l, uint32_t o) {
    repage_gather_unit<CAST, POW2, SCALED, PPOW2>(P, T, j, l, o, r, scales);
  });
}

// kvbm_gated_repage_gather_kernel over a batch of sequences (num_big: the length of `units`): layer l is done once it landed for
// every sequence.
template <int CAST, bool POW2, bool SCALED, bool PPOW2>
__global__ void __launch_bounds__(256)
kvbm_gated_batch_repage_gather_kernel(const __grid_constant__ RepageGatherParams P, const __grid_constant__ GateArgs A,
                                      const kvbm_repage_unit* units, uint32_t num_big, RowSplit r, const float* scales, uint32_t batch)
{
  gated_repage_units(A, P.g, P.geo, num_big, batch, [&](const GatherStage& T, uint32_t j, uint32_t l, uint32_t o) {
    repage_gather_unit<CAST, POW2, SCALED, PPOW2, kSeqs>(P, T, j, l, o, r, scales, units);
  });
}

// kvbm_gated_batch_repage_gather_kernel over a routed batch (num_big: the length of `routes`).  Each stage's sources are the
// routed ones only (the launch ANDs the union of the batch's masks in), so a source no sequence reads is never waited on.
template <int CAST, bool POW2, bool SCALED, bool PPOW2>
__global__ void __launch_bounds__(256, 1)
kvbm_gated_repage_fanin_kernel(const __grid_constant__ RepageGatherParams P, const __grid_constant__ GateArgs A, const __grid_constant__ SourceHeads H,
                               const kvbm_route_unit* routes, uint32_t num_big, RowSplit r, const float* scales, uint32_t batch)
{
  gated_repage_units(A, P.g, P.geo, num_big, batch, [&](const GatherStage& T, uint32_t j, uint32_t l, uint32_t o) {
    repage_gather_unit<CAST, POW2, SCALED, PPOW2, kRouted>(P, T, j, l, o, r, scales, routes, H.n);
  });
}

// kvbm_gated_batch_repage_gather_kernel over a batch whose pages need not divide (num_big: the length of `units`).
template <int CAST, bool POW2, bool SCALED, bool PPOW2>
__global__ void __launch_bounds__(256)
kvbm_gated_repage_anypage_kernel(const __grid_constant__ RepageGatherParams P, const __grid_constant__ GateArgs A,
                                 const kvbm_repage_anypage_unit* units, uint32_t num_big, RowSplit r, const float* scales, uint32_t batch)
{
  gated_repage_units(A, P.g, P.geo, num_big, batch, [&](const GatherStage& T, uint32_t j, uint32_t l, uint32_t o) {
    repage_gather_unit<CAST, POW2, SCALED, PPOW2, kPhased>(P, T, j, l, o, r, scales, units);
  });
}

// kvbm_gated_repage_fanin_kernel over a batch whose pages need not divide (num_big: the length of `units`): the stages' sources are
// the routed ones only, as there.
template <int CAST, bool POW2, bool SCALED, bool PPOW2>
__global__ void __launch_bounds__(256, 1)
kvbm_gated_repage_collect_kernel(const __grid_constant__ RepageGatherParams P, const __grid_constant__ GateArgs A,
                                 const __grid_constant__ SourceHeads H, const kvbm_route_anypage_unit* units, uint32_t num_big, RowSplit r,
                                 const float* scales, uint32_t batch)
{
  gated_repage_units(A, P.g, P.geo, num_big, batch, [&](const GatherStage& T, uint32_t j, uint32_t l, uint32_t o) {
    repage_gather_unit<CAST, POW2, SCALED, PPOW2, kRoutedPhased>(P, T, j, l, o, r, scales, units, H.n);
  });
}

// The push kernels' hook in arrive_transfer: the num_flags target done flags of F, with A.ss's own and before the completion word.
__device__ __forceinline__ auto target_done(const ScatterFlags& F, const int& num_flags, const GateArgs& A)
{
  return [&] {
    for (int t = 0; t < num_flags; ++t)
      if (F.done[t]) ptx::st_relaxed_sys(F.done[t], A.ss.epoch);
  };
}

// kvbm_paged_repage_scatter_kernel's unit walk behind the one source's gate; unit = (l * num_big + j) * no + o over the source
// layer range, so layer_done[l] counts source layer l in every target.
template <int CAST, bool POW2, bool SCALED, bool PPOW2>
__global__ void __launch_bounds__(256, 1)
kvbm_gated_repage_push_kernel(const __grid_constant__ ScatterParams P, const __grid_constant__ GateArgs A, const __grid_constant__ ScatterFlags F,
                              int num_flags, uint32_t num_big, RowSplit r, const float* scales, uint32_t batch)
{
  gated_repage_units(
      A, P, P.geo, num_big, batch,
      [&](const GatherStage& T, uint32_t j, uint32_t l, uint32_t o) { scatter_unit<CAST, POW2, SCALED, PPOW2>(P, T, j, l, o, r, scales); },
      target_done(F, num_flags, A));
}

// kvbm_gated_repage_push_kernel over a batch of sequences (num_big: the length of `units`): source layer l is done once it landed
// in every target for every sequence.
template <int CAST, bool POW2, bool SCALED, bool PPOW2>
__global__ void __launch_bounds__(256, 1)
kvbm_gated_repage_push_seqs_kernel(const __grid_constant__ ScatterParams P, const __grid_constant__ GateArgs A, const __grid_constant__ ScatterFlags F,
                                   int num_flags, const kvbm_repage_unit* units, uint32_t num_big, RowSplit r, const float* scales, uint32_t batch)
{
  gated_repage_units(
      A, P, P.geo, num_big, batch,
      [&](const GatherStage& T, uint32_t j, uint32_t l, uint32_t o) { scatter_unit<CAST, POW2, SCALED, PPOW2, kSeqs>(P, T, j, l, o, r, scales, units); },
      target_done(F, num_flags, A));
}

// kvbm_gated_repage_push_seqs_kernel over a routed batch (num_big: the length of `routes`): every unit of source layer l counts,
// written or not, so layer l is done once it landed in every target each sequence is routed to.
template <int CAST, bool POW2, bool SCALED, bool PPOW2>
__global__ void __launch_bounds__(256, 1)
kvbm_gated_repage_route_kernel(const __grid_constant__ ScatterParams P, const __grid_constant__ GateArgs A, const __grid_constant__ ScatterFlags F,
                               int num_flags, const kvbm_route_unit* routes, uint32_t num_big, RowSplit r, const float* scales, uint32_t batch)
{
  gated_repage_units(
      A, P, P.geo, num_big, batch,
      [&](const GatherStage& T, uint32_t j, uint32_t l, uint32_t o) {
        scatter_unit<CAST, POW2, SCALED, PPOW2, kRouted>(P, T, j, l, o, r, scales, routes);
      },
      target_done(F, num_flags, A));
}

// kvbm_gated_repage_push_seqs_kernel over a batch whose pages need not divide (num_big: the length of `units`).
template <int CAST, bool POW2, bool SCALED, bool PPOW2>
__global__ void __launch_bounds__(256, 1)
kvbm_gated_repage_phased_push_kernel(const __grid_constant__ ScatterParams P, const __grid_constant__ GateArgs A,
                                     const __grid_constant__ ScatterFlags F, int num_flags, const kvbm_repage_anypage_unit* units,
                                     uint32_t num_big, RowSplit r, const float* scales, uint32_t batch)
{
  gated_repage_units(
      A, P, P.geo, num_big, batch,
      [&](const GatherStage& T, uint32_t j, uint32_t l, uint32_t o) {
        scatter_unit<CAST, POW2, SCALED, PPOW2, kPhased>(P, T, j, l, o, r, scales, units);
      },
      target_done(F, num_flags, A));
}

// kvbm_gated_repage_route_kernel over a batch whose pages need not divide (num_big: the length of `units`): every unit of source
// layer l counts, written or not, as there.
template <int CAST, bool POW2, bool SCALED, bool PPOW2>
__global__ void __launch_bounds__(256, 1)
kvbm_gated_repage_deal_kernel(const __grid_constant__ ScatterParams P, const __grid_constant__ GateArgs A, const __grid_constant__ ScatterFlags F,
                              int num_flags, const kvbm_route_anypage_unit* units, uint32_t num_big, RowSplit r, const float* scales,
                              uint32_t batch)
{
  gated_repage_units(
      A, P, P.geo, num_big, batch,
      [&](const GatherStage& T, uint32_t j, uint32_t l, uint32_t o) {
        scatter_unit<CAST, POW2, SCALED, PPOW2, kRoutedPhased>(P, T, j, l, o, r, scales, units);
      },
      target_done(F, num_flags, A));
}

// The stream-wait form's signal after layer l: its layer-done flag, and after the last layer the done and completion flags.
__global__ void kvbm_layer_signal_kernel(uint32_t* layer_done, uint32_t* done, uint32_t epoch, uint32_t* completion, uint32_t completion_value)
{
  __threadfence_system();
  if (layer_done) ptx::st_release_sys(layer_done, epoch);
  if (done) ptx::st_release_sys(done, epoch);
  if (completion) ptx::st_release_sys(completion, completion_value);
}

// The instantiation of the permuting kernels a launch takes for its cast mode, row split and scales: calls
// f(integral_constant<int, CAST>, bool_constant<POW2>, bool_constant<SCALED>).  Scales without a cast take the unscaled
// instantiation (the launch rejects them first), so no scaled kernel exists without a cast.  preload_kernels() passes every
// run-time combination through here, so whatever a launch can pick is loaded up front.
template <class F>
static void with_walk_kernel(int cast_mode, bool pow2, bool scaled, F&& f)
{
  auto go = [&](auto cast, auto sc) { pow2 ? f(cast, std::true_type{}, sc) : f(cast, std::false_type{}, sc); };
  using Up = std::integral_constant<int, KVBM_CAST_FP8E4M3_TO_BF16>;
  using Down = std::integral_constant<int, KVBM_CAST_BF16_TO_FP8E4M3>;
  switch (cast_mode) {
    case KVBM_CAST_NONE: return go(std::integral_constant<int, KVBM_CAST_NONE>{}, std::false_type{});
    case KVBM_CAST_FP8E4M3_TO_BF16: return scaled ? go(Up{}, std::true_type{}) : go(Up{}, std::false_type{});
    default: return scaled ? go(Down{}, std::true_type{}) : go(Down{}, std::false_type{});
  }
}

// with_walk_kernel for the re-paging kernels, whose last template argument is the small page's split: calls
// f(cast, row pow2, scaled, bool_constant<PAGE_POW2>).
template <class F>
static void with_repage_kernel(int cast_mode, bool pow2, bool scaled, bool page_pow2, F&& f)
{
  with_walk_kernel(cast_mode, pow2, scaled, [&](auto c, auto p, auto sc) {
    page_pow2 ? f(c, p, sc, std::true_type{}) : f(c, p, sc, std::false_type{});
  });
}

// The one place that names each unit kind's kernels: the re-paging gather's and the scatter's one-CTA-per-unit kernel and gated
// kernel, the kind's sequence and unit record types and the exported helper that writes (and counts) its unit table.  The
// launchers and preload_kernels take every kernel from here.
template <RepageUnits UNITS>
struct RepageKernels;
#define KVBM_REPAGE_KERNELS(UNITS, SEQ, RECORD, WRITE_UNITS, GATHER, GATED_GATHER, SCATTER, GATED_SCATTER)      \
  template <>                                                                                                   \
  struct RepageKernels<UNITS> {                                                                                 \
    using Seq = SEQ;                                                                                            \
    using Record = RECORD;                                                                                      \
    static constexpr auto write_units = WRITE_UNITS;                                                            \
    template <int C, bool P, bool S, bool PP> static constexpr auto gather = GATHER<C, P, S, PP>;               \
    template <int C, bool P, bool S, bool PP> static constexpr auto gated_gather = GATED_GATHER<C, P, S, PP>;   \
    template <int C, bool P, bool S, bool PP> static constexpr auto scatter = SCATTER<C, P, S, PP>;             \
    template <int C, bool P, bool S, bool PP> static constexpr auto gated_scatter = GATED_SCATTER<C, P, S, PP>; \
  };
KVBM_REPAGE_KERNELS(kRange, void, void, nullptr, kvbm_paged_repage_gather_kernel, kvbm_gated_repage_gather_kernel,
                    kvbm_paged_repage_scatter_kernel, kvbm_gated_repage_push_kernel)
KVBM_REPAGE_KERNELS(kSeqs, kvbm_repage_seq, kvbm_repage_unit, kvbm_kernels_repage_batch_units, kvbm_paged_batch_repage_gather_kernel,
                    kvbm_gated_batch_repage_gather_kernel, kvbm_paged_repage_push_seqs_kernel, kvbm_gated_repage_push_seqs_kernel)
KVBM_REPAGE_KERNELS(kRouted, kvbm_route_seq, kvbm_route_unit, kvbm_kernels_repage_route_units, kvbm_paged_repage_fanin_kernel,
                    kvbm_gated_repage_fanin_kernel, kvbm_paged_repage_route_kernel, kvbm_gated_repage_route_kernel)
KVBM_REPAGE_KERNELS(kPhased, kvbm_repage_seq, kvbm_repage_anypage_unit, kvbm_kernels_repage_anypage_units, kvbm_paged_repage_anypage_kernel,
                    kvbm_gated_repage_anypage_kernel, kvbm_paged_repage_phased_push_kernel, kvbm_gated_repage_phased_push_kernel)
KVBM_REPAGE_KERNELS(kRoutedPhased, kvbm_route_seq, kvbm_route_anypage_unit, kvbm_kernels_repage_route_anypage_units,
                    kvbm_paged_repage_collect_kernel, kvbm_gated_repage_collect_kernel, kvbm_paged_repage_deal_kernel,
                    kvbm_gated_repage_deal_kernel)
#undef KVBM_REPAGE_KERNELS

// Calls f(integral_constant<RepageUnits, units>).
template <class F>
static void with_units(RepageUnits units, F&& f)
{
  switch (units) {
    case kRange: return f(std::integral_constant<RepageUnits, kRange>{});
    case kSeqs: return f(std::integral_constant<RepageUnits, kSeqs>{});
    case kRouted: return f(std::integral_constant<RepageUnits, kRouted>{});
    case kPhased: return f(std::integral_constant<RepageUnits, kPhased>{});
    case kRoutedPhased: return f(std::integral_constant<RepageUnits, kRoutedPhased>{});
  }
}

// with_repage_kernel with the unit kind first: calls f(integral_constant<RepageUnits, units>, cast, row pow2, scaled, page pow2).
template <class F>
static void with_repage_units(RepageUnits units, int cast_mode, bool pow2, bool scaled, bool page_pow2, F&& f)
{
  with_units(units, [&](auto u) {
    with_repage_kernel(cast_mode, pow2, scaled, page_pow2, [&](auto c, auto p, auto sc, auto pp) { f(u, c, p, sc, pp); });
  });
}

__global__ void kvbm_signal_kernel(uint32_t* a, uint32_t va, uint32_t* b, uint32_t vb)
{
  __threadfence_system();
  if (a) ptx::st_release_sys(a, va);
  if (b) ptx::st_release_sys(b, vb);
}

static size_t dtype_size(int dtype)
{
  switch (dtype) {
    case KVBM_DTYPE_F16:
    case KVBM_DTYPE_BF16:
      return 2;
    case KVBM_DTYPE_F32:
      return 4;
    case KVBM_DTYPE_F64:
      return 8;
    default:
      return 0;
  }
}

template <bool TO_UNIVERSAL>
static cudaError_t launch_permute(void* const* universal_ptrs, void* const* block_ptrs, size_t num_blocks,
                                  size_t nh, size_t nl, size_t no, size_t nt, size_t hd, int dtype,
                                  int layout, cudaStream_t stream)
{
  const size_t elem = dtype_size(dtype);
  if (elem == 0) return cudaErrorInvalidValue;  // tensor_kernels.cu:327
  const size_t total_per_block = nh * nl * no * nt * hd;
  if (total_per_block * num_blocks == 0) return cudaSuccess;  // tensor_kernels.cu:238-240
  if (!block_ptrs || !universal_ptrs) return cudaErrorInvalidValue;
  if (layout != KVBM_BLOCK_LAYOUT_NHD && layout != KVBM_BLOCK_LAYOUT_HND) return cudaErrorInvalidValue;
  if (total_per_block * elem >= (1ull << 32)) return cudaErrorInvalidValue;

  const size_t row = hd * elem;
  DeviceInfo di;
  cudaError_t e = device_info(&di);
  if (e != cudaSuccess) return e;
  RowSplit r;
  if (num_blocks * nl * no < (1ull << 31) && row_split(row, nt, &r)) {
    // the walk's strides: UniversalTP on the universal side, the chunk's own layout as an operational region
    kvbm_permute_side uni{}, chunk{};
    uni.kv_layout = KVBM_KV_UNIVERSAL_TP;
    chunk.kv_layout = layout == KVBM_BLOCK_LAYOUT_NHD ? KVBM_KV_OPERATIONAL_NHD : KVBM_KV_OPERATIONAL_HND;
    PermuteSide U, C;
    const uint32_t nl32 = static_cast<uint32_t>(nl), no32 = static_cast<uint32_t>(no), nh32 = static_cast<uint32_t>(nh),
                   nt32 = static_cast<uint32_t>(nt);
    fill_permute_side(uni, nl32, no32, nh32, nt32, static_cast<uint32_t>(row), &U);
    fill_permute_side(chunk, nl32, no32, nh32, nt32, static_cast<uint32_t>(row), &C);
    const PermuteSide& S = TO_UNIVERSAL ? C : U;
    const PermuteSide& D = TO_UNIVERSAL ? U : C;
    const unsigned grid = static_cast<unsigned>(num_blocks * nl * no);
    const int threads = static_cast<int>(std::min<size_t>(8, nh)) * 32;
    if (r.pow2)
      kvbm_permute_table_kernel<true><<<grid, threads, 0, stream>>>(universal_ptrs, block_ptrs, S, D, nl32, no32, nh32, nt32, r, static_cast<uint32_t>(elem));
    else
      kvbm_permute_table_kernel<false><<<grid, threads, 0, stream>>>(universal_ptrs, block_ptrs, S, D, nl32, no32, nh32, nt32, r, static_cast<uint32_t>(elem));
    g_launches.fetch_add(1, std::memory_order_relaxed);
    return cudaGetLastError();
  }
  // The vector must divide a head row AND every buffer must be aligned to it.  Chunk/universal
  // buffers come from cudaMalloc / torch (>= 256 B aligned) in practice, but the ABI takes raw
  // pointers, so only widen past the element size when the row allows it and keep 2/4/8-byte
  // vectors naturally aligned with the element type.
  int vec = static_cast<int>(elem);
  if (row % 16 == 0)
    vec = 16;
  else if (row % 8 == 0 && elem <= 8)
    vec = std::max<int>(vec, 8);
  else if (row % 4 == 0 && elem <= 4)
    vec = std::max<int>(vec, 4);
  const uint32_t hdv = static_cast<uint32_t>(row / vec);
  const uint32_t units_per_block = static_cast<uint32_t>(total_per_block * elem / vec);
  const uint64_t total_units = static_cast<uint64_t>(units_per_block) * num_blocks;
  const uint64_t want = (total_units + 255) / 256;
  const int grid = static_cast<int>(std::min<uint64_t>(want, static_cast<uint64_t>(di.sm_count) * 16));
  auto go = [&](auto kern) {
    kern<<<grid, 256, 0, stream>>>(universal_ptrs, block_ptrs, total_units, units_per_block,
                                   static_cast<uint32_t>(nh), static_cast<uint32_t>(nl),
                                   static_cast<uint32_t>(no), static_cast<uint32_t>(nt), hdv, layout);
  };
  switch (vec) {
    case 16: go(kvbm_permute_kernel<16, TO_UNIVERSAL>); break;
    case 8: go(kvbm_permute_kernel<8, TO_UNIVERSAL>); break;
    case 4: go(kvbm_permute_kernel<4, TO_UNIVERSAL>); break;
    default: go(kvbm_permute_kernel<2, TO_UNIVERSAL>); break;
  }
  g_launches.fetch_add(1, std::memory_order_relaxed);
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------
// tiny flag kernels
// ------------------------------------------------------------------------------------------------
__global__ void kvbm_set_flags_kernel(uint32_t* flags, int first, int count, uint32_t value)
{
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < count) {
    __threadfence_system();
    ptx::st_release_sys(flags + first + i, value);
  }
}
// The fallback of kvbm_kernels_wait_flag when stream memops are missing: the same cyclic order as CU_STREAM_WAIT_VALUE_GEQ.
__global__ void kvbm_wait_flag_kernel(const uint32_t* flag, uint32_t value)
{
  while (!epoch_reached(ptx::ld_acquire_sys(flag), value)) __nanosleep(100);
}

static cudaError_t preload_kernels()
{
  cudaFuncAttributes attr;
  cudaError_t e = cudaSuccess;
#define KVBM_PRELOAD(k) \
  if ((e = cudaFuncGetAttributes(&attr, k)) != cudaSuccess) return e;
  KVBM_PRELOAD(kvbm_pair_copy_kernel)
  KVBM_PRELOAD((kvbm_paged_copy_kernel<KVBM_CAST_NONE, false>))
  KVBM_PRELOAD((kvbm_paged_copy_kernel<KVBM_CAST_FP8E4M3_TO_BF16, false>))
  KVBM_PRELOAD((kvbm_paged_copy_kernel<KVBM_CAST_BF16_TO_FP8E4M3, false>))
  KVBM_PRELOAD((kvbm_paged_copy_kernel<KVBM_CAST_NONE, true>))
  KVBM_PRELOAD((kvbm_paged_copy_kernel<KVBM_CAST_FP8E4M3_TO_BF16, true>))
  KVBM_PRELOAD((kvbm_paged_copy_kernel<KVBM_CAST_BF16_TO_FP8E4M3, true>))
  KVBM_PRELOAD((kvbm_paged_copy_kernel<KVBM_CAST_FP8E4M3_TO_BF16, false, true>))
  KVBM_PRELOAD((kvbm_paged_copy_kernel<KVBM_CAST_BF16_TO_FP8E4M3, false, true>))
  KVBM_PRELOAD(kvbm_set_flags_kernel)
  KVBM_PRELOAD(kvbm_wait_flag_kernel)
  KVBM_PRELOAD(kvbm_signal_kernel)
  KVBM_PRELOAD(kvbm_permute_table_kernel<true>)
  KVBM_PRELOAD(kvbm_permute_table_kernel<false>)
  KVBM_PRELOAD((kvbm_permute_kernel<16, true>))
  KVBM_PRELOAD((kvbm_permute_kernel<8, true>))
  KVBM_PRELOAD((kvbm_permute_kernel<4, true>))
  KVBM_PRELOAD((kvbm_permute_kernel<2, true>))
  KVBM_PRELOAD((kvbm_permute_kernel<16, false>))
  KVBM_PRELOAD((kvbm_permute_kernel<8, false>))
  KVBM_PRELOAD((kvbm_permute_kernel<4, false>))
  KVBM_PRELOAD((kvbm_permute_kernel<2, false>))
#undef KVBM_PRELOAD
  // the paged permute, the gather and the plain re-page: every instantiation their launchers can select, through their own
  // selection helpers
  for (int cast = KVBM_CAST_NONE; cast <= KVBM_CAST_BF16_TO_FP8E4M3; ++cast)
    for (int pow2 = 0; pow2 < 2; ++pow2)
      for (int scaled = 0; scaled < 2; ++scaled)
        with_walk_kernel(cast, pow2, scaled, [&](auto c, auto p, auto sc) {
          if (e == cudaSuccess) e = cudaFuncGetAttributes(&attr, kvbm_paged_permute_kernel<c, p, sc>);
          if (e == cudaSuccess) e = cudaFuncGetAttributes(&attr, kvbm_paged_gather_kernel<c, p, sc>);
          if (e == cudaSuccess) e = cudaFuncGetAttributes(&attr, kvbm_paged_repage_kernel<c, p, sc, true>);
          if (e == cudaSuccess) e = cudaFuncGetAttributes(&attr, kvbm_paged_repage_kernel<c, p, sc, false>);
          if (e == cudaSuccess) e = cudaFuncGetAttributes(&attr, kvbm_gated_gather_kernel<c, p, sc>);
        });
  // the re-paging gathers and scatters: every kernel of every unit kind (RepageKernels)
  for (int units = kRange; units <= kRoutedPhased; ++units)
    for (int cast = KVBM_CAST_NONE; cast <= KVBM_CAST_BF16_TO_FP8E4M3; ++cast)
      for (int pow2 = 0; pow2 < 2; ++pow2)
        for (int scaled = 0; scaled < 2; ++scaled)
          for (int page_pow2 = 0; page_pow2 < 2; ++page_pow2)
            with_repage_units(static_cast<RepageUnits>(units), cast, pow2, scaled, page_pow2, [&](auto u, auto c, auto p, auto sc, auto pp) {
              using K = RepageKernels<u>;
              if (e == cudaSuccess) e = cudaFuncGetAttributes(&attr, K::template gather<c, p, sc, pp>);
              if (e == cudaSuccess) e = cudaFuncGetAttributes(&attr, K::template gated_gather<c, p, sc, pp>);
              if (e == cudaSuccess) e = cudaFuncGetAttributes(&attr, K::template scatter<c, p, sc, pp>);
              if (e == cudaSuccess) e = cudaFuncGetAttributes(&attr, K::template gated_scatter<c, p, sc, pp>);
            });
  if (e == cudaSuccess) e = cudaFuncGetAttributes(&attr, kvbm_layer_signal_kernel);
  if (e == cudaSuccess) e = cudaFuncGetAttributes(&attr, kvbm_scatter_signal_kernel);
  return e;
}

// Stream memory operations (cuStreamWriteValue32 / cuStreamWaitValue32) through the driver entry point:
// the stream's front-end writes / polls the word itself -- no kernel launch, no SM occupied by a spinner.
typedef int (*stream_memop_fn)(cudaStream_t, unsigned long long, uint32_t, unsigned int);
static stream_memop_fn g_write32 = nullptr, g_wait32 = nullptr;
static std::atomic<int> g_memops_state{0};  // 0 unknown, 1 available, -1 unavailable

static bool stream_memops()
{
  int st = g_memops_state.load(std::memory_order_acquire);
  if (st == 0) {
    void *w = nullptr, *q = nullptr;
    cudaDriverEntryPointQueryResult r1, r2;
    bool ok = cudaGetDriverEntryPoint("cuStreamWriteValue32", &w, cudaEnableDefault, &r1) == cudaSuccess && w &&
              cudaGetDriverEntryPoint("cuStreamWaitValue32", &q, cudaEnableDefault, &r2) == cudaSuccess && q;
    (void)cudaGetLastError();
    g_write32 = reinterpret_cast<stream_memop_fn>(w);
    g_wait32 = reinterpret_cast<stream_memop_fn>(q);
    st = ok ? 1 : -1;
    g_memops_state.store(st, std::memory_order_release);
  }
  return st == 1;
}

template <class K>
static cudaError_t set_smem(K kernel, uint32_t bytes)
{
  return cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(bytes));
}

// The launch checks every permuting and re-paging entry shares.  Before the empty-range signal: a cast mode the walk knows, and
// scales only with a cast (they belong to the fp8 side of it).
static bool cast_args_ok(int cast_mode, const float* cast_scales)
{
  if (cast_mode < KVBM_CAST_NONE || cast_mode > KVBM_CAST_BF16_TO_FP8E4M3) return false;
  return !(cast_scales && cast_mode == KVBM_CAST_NONE);
}

// The signal launch after the work (or instead of it on an empty range): done_flag / completion_flag written once.
static cudaError_t signal_launch(uint32_t* done_flag, uint32_t epoch, uint32_t* completion_flag, uint32_t completion_value, cudaStream_t stream)
{
  if (!done_flag && !completion_flag) return cudaSuccess;
  kvbm_signal_kernel<<<1, 1, 0, stream>>>(done_flag, epoch, completion_flag, completion_value);
  g_launches.fetch_add(1, std::memory_order_relaxed);
  return cudaGetLastError();
}

// The end of a transform's launch: count it, and return its launch error or, on success, the signal launch's.
static cudaError_t launched(cudaStream_t stream, uint32_t* done_flag = nullptr, uint32_t epoch = 0, uint32_t* completion_flag = nullptr,
                            uint32_t completion_value = 0)
{
  g_launches.fetch_add(1, std::memory_order_relaxed);
  const cudaError_t e = cudaGetLastError();
  return e != cudaSuccess ? e : signal_launch(done_flag, epoch, completion_flag, completion_value, stream);
}

// The walk splits the fp8 side's row into 16 B vectors when casting (the bf16 side's vectors are 32 B), else the row; an odd
// bf16 row has no fp8 row.  Fills the destination's row and the row the walk counts vectors of.
static bool cast_rows(uint32_t src_row_bytes, int cast_mode, uint64_t* dst_row_bytes, uint64_t* walk_row)
{
  if (cast_mode == KVBM_CAST_BF16_TO_FP8E4M3 && (src_row_bytes & 1)) return false;
  *dst_row_bytes = cast_mode == KVBM_CAST_FP8E4M3_TO_BF16   ? 2ull * src_row_bytes
                   : cast_mode == KVBM_CAST_BF16_TO_FP8E4M3 ? src_row_bytes / 2
                                                            : src_row_bytes;
  *walk_row = cast_mode == KVBM_CAST_BF16_TO_FP8E4M3 ? *dst_row_bytes : src_row_bytes;
  return true;
}

// One source of a gather into a destination of dst_num_heads heads, outer_dim no and strides D: its table, its outer dims, its
// window inside both sides' heads, its region page * its heads * row and its strides over its own src_nl layers.  Fills *G but
// G->first.
static bool fill_gather_source(const kvbm_permute_source& X, uint32_t src_nl, uint32_t dst_num_heads, uint32_t no, uint32_t page_size,
                               uint32_t src_row_bytes, const PermuteSide& D, GatherSource* G)
{
  if (!X.side.block_ids || !X.side.layout.layer_base || X.side.layout.outer_dim != no) return false;
  if (X.head_count == 0 || static_cast<uint64_t>(X.src_head_begin) + X.head_count > X.num_heads ||
      static_cast<uint64_t>(X.dst_head_begin) + X.head_count > dst_num_heads)
    return false;
  if (static_cast<uint64_t>(page_size) * X.num_heads * src_row_bytes != X.side.layout.region_bytes) return false;
  if (!fill_permute_side(X.side, src_nl, no, X.num_heads, page_size, src_row_bytes, &G->S)) return false;
  G->s_win = X.src_head_begin * G->S.head_stride;  // the windows' first heads
  G->d_win = X.dst_head_begin * D.head_stride;
  return true;
}

static bool heads_overlap(const kvbm_permute_source& a, const kvbm_permute_source& b)
{
  return a.dst_head_begin < b.dst_head_begin + b.head_count && b.dst_head_begin < a.dst_head_begin + a.head_count;
}

// The stage of layer window [begin, end) (a gather's destination layers, the scatter's source layers) among T[0 .. *num_stages):
// an equal window's, else a new one without sources; -1 when the window partly overlaps a stage.
static int window_stage(GatherStage* T, int* num_stages, uint32_t begin, uint32_t end)
{
  int k = 0;
  while (k < *num_stages && !(T[k].begin == begin && T[k].end == end)) {
    if (begin < T[k].end && T[k].begin < end) return -1;  // a partial overlap
    ++k;
  }
  if (k == *num_stages) T[(*num_stages)++] = GatherStage{begin, end, 0, 0, 0};
  return k;
}

// order[i]: the i-th of window_stage's stages in ascending layers (an insertion sort of at most 16); whether they tile [lb, le).
static bool order_stages(const GatherStage* T, int num_stages, int lb, int le, int* order)
{
  for (int k = 0; k < num_stages; ++k) {
    int at = k;
    while (at > 0 && T[order[at - 1]].begin > T[k].begin) {
      order[at] = order[at - 1];
      --at;
    }
    order[at] = k;
  }
  uint32_t reached = static_cast<uint32_t>(lb);
  for (int i = 0; i < num_stages; ++i)
    if (T[order[i]].begin <= reached && T[order[i]].end > reached) reached = T[order[i]].end;
  return reached >= static_cast<uint32_t>(le);
}

// The sources of a gather into P->D (nl layers, dst_num_heads heads) over destination layers [lb, le): each layer window
// non-empty and inside its source's own layers and the destination's; two windows equal (one stage) or disjoint in the
// destination; the stages covering every layer of [lb, le); within a stage, windows on destination heads no other window of the
// stage writes (two would race); every rule of fill_gather_source; at most max_covered covered heads over all stages.  Fills
// P->src, P->covered, P->stage and P->shift, and with several sources the head map P->entry, stage by stage in ascending
// destination layers; *widest: the most heads of one stage.  masks: a routed gather's distinct source masks, under which two
// windows of a stage may share destination heads unless one mask holds both.
static bool fill_stage_sources(const kvbm_stage_source* srcs, int num_srcs, uint32_t dst_num_heads, uint32_t nl, uint32_t no, int lb, int le,
                               uint32_t page_size, uint32_t src_row_bytes, uint32_t max_covered, GatherParams* P, uint32_t* widest,
                               const std::vector<uint32_t>* masks = nullptr)
{
  int stage_of_src[KVBM_GATHER_MAX_SOURCES];
  int num_stages = 0;
  GatherStage* T = P->stage;
  auto routed_together = [&](int s, int t) {
    if (!masks) return true;
    for (uint32_t m : *masks)
      if (((m >> s) & 1u) && ((m >> t) & 1u)) return true;
    return false;
  };
  for (int s = 0; s < num_srcs; ++s) {
    const kvbm_stage_source& X = srcs[s];
    const uint64_t src_end = static_cast<uint64_t>(X.src_layer_begin) + X.layer_count, dst_end = static_cast<uint64_t>(X.dst_layer_begin) + X.layer_count;
    if (X.layer_count == 0 || src_end > X.src.side.layout.num_layers || dst_end > nl) return false;
    const int k = stage_of_src[s] = window_stage(T, &num_stages, X.dst_layer_begin, static_cast<uint32_t>(dst_end));
    if (k < 0) return false;
    for (int t = 0; t < s; ++t)
      if (stage_of_src[t] == k && heads_overlap(X.src, srcs[t].src) && routed_together(s, t)) return false;
    T[k].sources |= 1u << s;
    P->shift[s] = X.src_layer_begin - X.dst_layer_begin;
  }
  int order[KVBM_GATHER_MAX_SOURCES];
  if (!order_stages(T, num_stages, lb, le, order)) return false;
  GatherStage sorted[KVBM_GATHER_MAX_SOURCES] = {};
  uint32_t covered = 0;
  *widest = 0;
  for (int i = 0; i < num_stages; ++i) {
    GatherStage& S = sorted[i] = T[order[i]];
    S.first = covered;
    for (int s = 0; s < num_srcs; ++s) {
      if (!((S.sources >> s) & 1u)) continue;
      const kvbm_permute_source& X = srcs[s].src;
      GatherSource& G = P->src[s];
      if (!fill_gather_source(X, X.side.layout.num_layers, dst_num_heads, no, page_size, src_row_bytes, P->D, &G)) return false;
      if (static_cast<uint64_t>(covered) + X.head_count > max_covered) return false;
      G.first = covered;
      if (num_srcs > 1)
        for (uint32_t j = 0; j < X.head_count; ++j) P->entry[covered + j] = static_cast<uint8_t>(s);
      covered += X.head_count;
    }
    S.count = covered - S.first;
    *widest = std::max(*widest, S.count);
  }
  std::copy(sorted, sorted + KVBM_GATHER_MAX_SOURCES, T);
  P->covered = covered;
  return true;
}

// The gate's own argument rules (kvbm_permute_stream), checked before anything else of a streamed entry: a descriptor, a known
// gate mode, a workspace when the caller asks for the spinning form, and a ready-flag array for every used source (a routed
// gather's: every source of `used`).
static bool stream_args_ok(const kvbm_permute_stream* st, int num_srcs, uint32_t used = ~0u)
{
  if (!st || st->gate_mode < KVBM_GATE_AUTO || st->gate_mode > KVBM_GATE_STREAM_WAIT) return false;
  if (st->gate_mode == KVBM_GATE_SPIN && !st->sync_workspace) return false;
  for (int s = 0; s < num_srcs && s < KVBM_GATHER_MAX_SOURCES; ++s)
    if (((used >> s) & 1u) && !st->layer_ready_flags[s]) return false;
  return true;
}

// The form of a streamed launch, after every argument check: 1 spinning, 2 stream-wait (kvbm_paged_copy_v2's rule for gate_mode),
// 0 with *err set when neither can run.  Loads every kernel of the library first (device_info), as the paged copy's gate does.
static int gate_form(const kvbm_permute_stream& st, cudaError_t* err)
{
  DeviceInfo di;
  if ((*err = device_info(&di)) != cudaSuccess) return 0;
  bool spin = st.gate_mode == KVBM_GATE_SPIN || (st.gate_mode == KVBM_GATE_AUTO && eager_module_loading());
  if (!spin && !stream_memops()) {
    if (st.gate_mode != KVBM_GATE_AUTO) {
      *err = cudaErrorNotSupported;
      return 0;
    }
    spin = true;
  }
  if (spin && !st.sync_workspace) {  // AUTO chose the spinning form, whose abort word and counters live in the workspace
    *err = cudaErrorInvalidValue;
    return 0;
  }
  return spin ? 1 : 2;
}

// The spinning form's default grid: half the SMs.  A spinning CTA holds its SM for the whole prefill, and an SM that already runs
// a CTA of one kernel does not always take a CTA of another (a shared-memory carveout of its own, for one): with a spinning CTA
// on every SM of an H100 a producer's one-thread layer kernel never started and the gate timed out.  Half the SMs leaves the
// engine at least as many SMs as the transfer holds, wherever the CTAs are placed.
static int gate_default_ctas(const DeviceInfo& di) { return std::max(1, di.sm_count / 2); }

// The spinning form's grid (max_ctas, 0 = gate_default_ctas, never more CTAs than units), its batch (units per ticket: about
// half a CTA's share of a layer, 1 .. 8) and its StreamSync: the workspace's [nl] layer counters and 3 control words, the units
// of one layer per layer, the destination's flags as the one flag destination.
static cudaError_t gate_args(const kvbm_permute_stream& st, int num_srcs, uint32_t nl, int layer_begin, int layer_end, uint64_t units,
                             GateArgs* A, unsigned* grid, uint32_t* batch)
{
  DeviceInfo di;
  cudaError_t e = device_info(&di);
  if (e != cudaSuccess) return e;
  const int cap = st.max_ctas > 0 ? st.max_ctas : gate_default_ctas(di);
  *grid = static_cast<unsigned>(std::min<uint64_t>(units, static_cast<uint64_t>(cap)));
  const uint64_t per_layer = units / static_cast<uint64_t>(layer_end - layer_begin);
  *batch = static_cast<uint32_t>(std::min<uint64_t>(8, std::max<uint64_t>(1, (per_layer + 2ull * *grid - 1) / (2ull * *grid))));
  *A = GateArgs{};
  StreamSync& ss = A->ss;
  ss.gate = true;
  ss.layer_counters = st.sync_workspace;
  ss.ctl = st.sync_workspace + nl;
  ss.done_flag[0] = st.done_flag;
  ss.layer_done[0] = st.layer_done_flags;
  ss.completion_flag = st.completion_flag;
  ss.completion_value = st.completion_value;
  ss.epoch = st.epoch;
  ss.total_rings = *grid;
  ss.items_per_layer = static_cast<uint32_t>(units / static_cast<uint64_t>(layer_end - layer_begin));
  ss.ndst = 1;
  ss.layer_begin = layer_begin;
  ss.layer_end = layer_end;
  ss.gate_timeout_ns = static_cast<uint64_t>(st.gate_timeout_ms > 0 ? st.gate_timeout_ms : 10000) * 1000000ull;
  ss.want_layers = st.layer_done_flags != nullptr;
  ss.want_done = st.done_flag != nullptr || st.completion_flag != nullptr;
  for (int s = 0; s < num_srcs; ++s) A->ready[s] = st.layer_ready_flags[s];
  A->num_ready = num_srcs;
  return cudaSuccess;
}

// A streamed launch of `units` units over layers [layer_begin, layer_end) of an nl-layer launch (a gather's destination, the
// scatter's source), after every argument check.  The spinning form: launch_gated(A, ctas, batch) launches the gated kernel,
// which writes every flag itself.  The stream-wait form: per layer l, the stream waits for the flag of every source of l's stage
// in P (a gather's or a scatter's) at the source's own layer (cuStreamWaitValue32, GEQ: the cyclic order of epoch_reached),
// launch_layer(l) moves the layer (unsignalled, but for a scatter's target flags after its last layer), and one signal launch
// writes its layer-done flag, plus the done and completion flags after the last layer.  Nothing resident spins.
template <class Params, class Layer, class Gated>
static cudaError_t launch_streamed(const kvbm_permute_stream& st, const Params& P, int num_srcs, uint32_t nl, int layer_begin,
                                   int layer_end, uint64_t units, cudaStream_t stream, Layer&& launch_layer, Gated&& launch_gated)
{
  cudaError_t e;
  const int form = gate_form(st, &e);
  if (form == 0) return e;
  if (form == 1) {
    GateArgs A;
    unsigned ctas;
    uint32_t batch;
    if ((e = gate_args(st, num_srcs, nl, layer_begin, layer_end, units, &A, &ctas, &batch)) != cudaSuccess) return e;
    launch_gated(A, ctas, batch);
    return launched(stream);
  }
  for (int l = layer_begin; l < layer_end; ++l) {
    const uint32_t mask = stage_of(P, static_cast<uint32_t>(l)).sources;
    for (int s = 0; s < num_srcs; ++s) {
      if (!((mask >> s) & 1u)) continue;
      const uint32_t* flag = st.layer_ready_flags[s] + source_layer(P, s, static_cast<uint32_t>(l));
      if (g_wait32(stream, reinterpret_cast<unsigned long long>(flag), st.epoch, 0) != 0) return cudaErrorUnknown;
    }
    if ((e = launch_layer(l)) != cudaSuccess) return e;
    const bool last = l + 1 == layer_end;
    uint32_t* done = last ? st.done_flag : nullptr;
    uint32_t* completion = last ? st.completion_flag : nullptr;
    uint32_t* layer_done = st.layer_done_flags ? st.layer_done_flags + l : nullptr;
    if (layer_done || done || completion) {
      kvbm_layer_signal_kernel<<<1, 1, 0, stream>>>(layer_done, done, st.epoch, completion, st.completion_value);
      if ((e = launched(stream)) != cudaSuccess) return e;
    }
  }
  return cudaSuccess;
}

// A source that moves its own layers, all nl of the destination's: its layer window is the identity over them (a PP1 plan).
static bool whole_layers(const kvbm_stage_source& X, uint32_t nl)
{
  return X.src_layer_begin == 0 && X.dst_layer_begin == 0 && X.layer_count == nl && X.src.side.layout.num_layers == nl;
}

// The sources of an entry without layer windows in out[]: one stage over every layer of dst, every shift 0.  The gather's rule
// that each source has the destination's num_layers stays: a source without gets an empty window, which fill_stage_sources
// rejects.  A null srcs or a num_srcs outside 1 .. KVBM_GATHER_MAX_SOURCES gives null, which the launch rejects.
static const kvbm_stage_source* one_stage(const kvbm_permute_source* srcs, int num_srcs, const kvbm_permute_side* dst, kvbm_stage_source* out)
{
  if (!srcs || num_srcs < 1 || num_srcs > KVBM_GATHER_MAX_SOURCES) return nullptr;
  const uint32_t nl = dst ? dst->layout.num_layers : 0;
  for (int s = 0; s < num_srcs; ++s) out[s] = kvbm_stage_source{srcs[s], 0, 0, srcs[s].side.layout.num_layers == nl ? nl : 0};
  return out;
}

// Every permuting launch: a head transform is one source, a gather several, each with a layer window.  Runs the checks of every
// entry once, signals when there is nothing to move, and launches kvbm_paged_permute_kernel for one source over its whole layers
// (the faster of the two, DESIGN §4.2b) or else kvbm_paged_gather_kernel.  max_covered: how many destination heads the sources
// may cover together; at most KVBM_GATHER_MAX_HEADS (the gather's head map) unless the launch is the permute kernel's.  st: a
// streamed launch (its flags are the ones passed), which takes the gated gather kernel, or per layer this launch unstreamed.
static cudaError_t launch_paged_permute(const kvbm_stage_source* srcs, int num_srcs, const kvbm_permute_side* dst, uint32_t dst_num_heads,
                                        int num_blocks, int layer_begin, int layer_end, uint32_t page_size, uint32_t src_row_bytes,
                                        int cast_mode, const float* cast_scales, uint32_t* done_flag, uint32_t epoch,
                                        uint32_t* completion_flag, uint32_t completion_value, uint32_t max_covered, cudaStream_t stream,
                                        const kvbm_permute_stream* st = nullptr)
{
  if (num_blocks < 0 || layer_begin < 0 || layer_end < layer_begin) return cudaErrorInvalidValue;
  if (!cast_args_ok(cast_mode, cast_scales)) return cudaErrorInvalidValue;
  if (!srcs || num_srcs < 1 || num_srcs > KVBM_GATHER_MAX_SOURCES) return cudaErrorInvalidValue;
  if (num_blocks == 0 || layer_end == layer_begin) return signal_launch(done_flag, epoch, completion_flag, completion_value, stream);
  if (!dst || !dst->block_ids || !dst->layout.layer_base) return cudaErrorInvalidValue;
  const uint32_t nl = dst->layout.num_layers, no = dst->layout.outer_dim;
  if (nl == 0 || no == 0 || static_cast<uint32_t>(layer_end) > nl) return cudaErrorInvalidValue;
  uint64_t dst_row_bytes, walk_row;
  if (!cast_rows(src_row_bytes, cast_mode, &dst_row_bytes, &walk_row)) return cudaErrorInvalidValue;
  RowSplit r;
  if (page_size == 0 || !row_split(walk_row, page_size, &r)) return cudaErrorInvalidValue;
  if (static_cast<uint64_t>(page_size) * dst_num_heads * dst_row_bytes != dst->layout.region_bytes) return cudaErrorInvalidValue;
  GatherParams P{};
  if (!fill_permute_side(*dst, nl, no, dst_num_heads, page_size, static_cast<uint32_t>(dst_row_bytes), &P.D)) return cudaErrorInvalidValue;
  uint32_t widest;
  if (!fill_stage_sources(srcs, num_srcs, dst_num_heads, nl, no, layer_begin, layer_end, page_size, src_row_bytes, max_covered, &P, &widest))
    return cudaErrorInvalidValue;
  const uint64_t units = static_cast<uint64_t>(num_blocks) * (layer_end - layer_begin) * no;
  if (units >= (1ull << 31)) return cudaErrorInvalidValue;
  const int threads = static_cast<int>(std::min<uint32_t>(8, widest)) * 32;
  const unsigned grid = static_cast<unsigned>(units);
  const uint32_t lb = static_cast<uint32_t>(layer_begin), nlay = static_cast<uint32_t>(layer_end - layer_begin);
  if (st)
    return launch_streamed(
        *st, P, num_srcs, nl, layer_begin, layer_end, units, stream,
        [&](int l) {
          return launch_paged_permute(srcs, num_srcs, dst, dst_num_heads, num_blocks, l, l + 1, page_size, src_row_bytes, cast_mode,
                                      cast_scales, nullptr, 0, nullptr, 0, max_covered, stream);
        },
        [&](const GateArgs& A, unsigned ctas, uint32_t batch) {
          with_walk_kernel(cast_mode, r.pow2, cast_scales != nullptr, [&](auto c, auto p, auto sc) {
            kvbm_gated_gather_kernel<c, p, sc><<<ctas, threads, 0, stream>>>(P, A, static_cast<uint32_t>(num_blocks), lb, nlay, no, page_size,
                                                                             r, cast_scales, batch);
          });
        });
  with_walk_kernel(cast_mode, r.pow2, cast_scales != nullptr, [&](auto c, auto p, auto sc) {
    const GatherSource& G = P.src[0];
    if (num_srcs == 1 && whole_layers(srcs[0], nl))
      kvbm_paged_permute_kernel<c, p, sc><<<grid, threads, 0, stream>>>(G.S, P.D, lb, nlay, no, P.covered, page_size, r, G.s_win, G.d_win,
                                                                        cast_scales);
    else
      kvbm_paged_gather_kernel<c, p, sc><<<grid, threads, 0, stream>>>(P, lb, nlay, no, page_size, r, cast_scales);
  });
  return launched(stream, done_flag, epoch, completion_flag, completion_value);
}

// The page split's exactness bound (big_page + small_page - gcd) * small_page < 2^32.  The small side splits phase + q with
// q < big_page and phase a multiple of the gcd below small_page (0 when the pages divide), so phase + q < big + small - gcd.  The
// multiply-high with m = ceil(2^32 / small) = (2^32 + e) / small, e < small, is exact for every x with x * e < 2^32, which the
// bound gives.  When small_page divides big_page it reads big_page * small_page < 2^32.  A small page of 2^16 or more fails it
// (the factor big + small - gcd is at least big >= small), which keeps the 64-bit product from wrapping.
static bool repage_exact(uint64_t big_page, uint64_t small_page)
{
  return small_page < (1u << 16) && (big_page + small_page - std::gcd(big_page, small_page)) * small_page < (1ull << 32);
}

// What every re-paging launch derives from its two pages, and their checks: non-zero pages, one dividing the other unless
// `any` (kvbm_kernels_paged_stage_repage_gather_anypage), repage_exact, the cast's rows and the row split of the larger page.
// Fills everything of *G but the token range's fields and nh, the walk's row split, the destination's row and whether the small
// page is a power of two.
static bool repage_pages(uint32_t src_page, uint32_t dst_page, int layer_begin, int layer_end, uint32_t no, uint32_t src_row_bytes,
                         int cast_mode, RepageGeom* G, RowSplit* r, uint64_t* dst_row_bytes, bool* page_pow2, bool any = false)
{
  if (src_page == 0 || dst_page == 0) return false;
  const bool src_small = src_page < dst_page;
  const uint32_t big_page = src_small ? dst_page : src_page, small_page = src_small ? src_page : dst_page;
  if (!any && big_page % small_page) return false;
  if (!repage_exact(big_page, small_page)) return false;
  uint64_t walk_row;
  if (!cast_rows(src_row_bytes, cast_mode, dst_row_bytes, &walk_row) || !row_split(walk_row, big_page, r)) return false;
  RepageGeom g{};
  g.small_page = small_page;
  g.big_page = big_page;
  g.ratio = big_page / small_page;
  g.layer_begin = static_cast<uint32_t>(layer_begin);
  g.nlayers = static_cast<uint32_t>(layer_end - layer_begin);
  g.no = no;
  g.src_small = src_small ? 1 : 0;
  // the small page's split, in RowSplit's form: log2 of the page, or the page and ceil(2^32 / page)
  *page_pow2 = (small_page & (small_page - 1)) == 0;
  if (*page_pow2) {
    while ((1u << g.page.vpr) < small_page) ++g.page.vpr;
    g.page.pow2 = true;
  } else {
    g.page = {small_page, static_cast<uint32_t>(((1ull << 32) + small_page - 1) / small_page), false};
  }
  *G = g;
  return true;
}

// A batch of sequences of a re-paging launch: its unit kind (never kRange), the caller's ranges (host; RepageKernels<kind>::Seq,
// which for a routed kind carries each sequence's mask: a scatter's targets, a gather's sources) and the unit table of
// RepageKernels<kind>::Record (device-accessible).  repage_batch builds one from pointers of those types, batch_table reads
// the table back as one.
struct RepageBatch {
  RepageUnits kind;
  const void* seqs;
  size_t num_seqs;
  const void* table;
  size_t num_units;
};
template <RepageUnits UNITS>
static RepageBatch repage_batch(const typename RepageKernels<UNITS>::Seq* seqs, size_t num_seqs,
                                const typename RepageKernels<UNITS>::Record* table, size_t num_units)
{
  RepageBatch B;
  B.kind = UNITS;
  B.seqs = seqs;
  B.num_seqs = num_seqs;
  B.table = table;
  B.num_units = num_units;
  return B;
}
template <RepageUnits UNITS>
static auto batch_table(const RepageBatch* B) { return static_cast<const typename RepageKernels<UNITS>::Record*>(B->table); }

// What repage_launch derives: repage_pages' results with the token range's fields, the units to launch (0: nothing to move), the
// big blocks per (layer, outer), and the layers and outer dim of the pool whose layers the launch counts.
struct RepageLaunch {
  RepageGeom geo;
  RowSplit r;
  uint64_t dst_row_bytes, units;
  uint32_t num_big, nl, no;
  bool page_pow2;
};

// Every re-paging launch's first checks, before any CUDA call: ranges not reversed, cast_args_ok, and B checked by its kind's unit
// table helper (RepageKernels) with the caller's unit count; a phased kind takes repage_pages without the divisibility rule.  An
// empty range or batch then leaves L->units 0 (the caller signals).  Else `side` (a gather's destination, the scatter's source) needs a table, a base, a non-zero outer dim and the layer
// range; the pages repage_pages' rules; a single range slots in 32 bits (its last block of the larger page ends below 2^32); the
// launch fewer than 2^31 units.  False: rejected.
static bool repage_launch(const kvbm_permute_side* side, uint32_t src_page, uint32_t dst_page, uint32_t token_begin, uint32_t token_end,
                          int layer_begin, int layer_end, uint32_t src_row_bytes, int cast_mode, const float* cast_scales, const RepageBatch* B,
                          RepageLaunch* L)
{
  if (layer_begin < 0 || layer_end < layer_begin || (!B && token_end < token_begin)) return false;
  if (!cast_args_ok(cast_mode, cast_scales)) return false;
  size_t num_big = 0;
  if (B) {
    size_t src_ids, dst_ids;
    int bad = 1;
    with_units(B->kind, [&](auto u) {
      using K = RepageKernels<u>;
      if constexpr (u != kRange)
        bad = K::write_units(static_cast<const typename K::Seq*>(B->seqs), B->num_seqs, src_page, dst_page, nullptr, 0, &num_big, &src_ids,
                            &dst_ids);
    });
    if (bad || num_big != B->num_units || (num_big != 0 && !B->table)) return false;
  }
  L->units = 0;
  if ((B ? num_big == 0 : token_end == token_begin) || layer_end == layer_begin) return true;
  if (!side || !side->block_ids || !side->layout.layer_base) return false;
  const uint32_t nl = L->nl = side->layout.num_layers, no = L->no = side->layout.outer_dim;
  if (nl == 0 || no == 0 || static_cast<uint32_t>(layer_end) > nl) return false;
  RepageGeom& g = L->geo;
  if (!repage_pages(src_page, dst_page, layer_begin, layer_end, no, src_row_bytes, cast_mode, &g, &L->r, &L->dst_row_bytes, &L->page_pow2,
                    B && phased_units(B->kind)))
    return false;
  if (!B) {
    const uint64_t big_end = (static_cast<uint64_t>(token_end) + g.big_page - 1) / g.big_page * g.big_page;
    if (big_end >= (1ull << 32)) return false;
    g.big_first = token_begin / g.big_page;
    g.small_first = token_begin / g.small_page;
    g.token_begin = token_begin;
    g.token_end = token_end;
    num_big = static_cast<size_t>(big_end / g.big_page) - g.big_first;
  }
  if (num_big >= (1ull << 31) || (L->units = static_cast<uint64_t>(num_big) * g.nlayers) >= (1ull << 31) || (L->units *= no) >= (1ull << 31))
    return false;
  L->num_big = static_cast<uint32_t>(num_big);
  return true;
}

// Every re-paging launch: a plain re-page is one source whose window covers every head and every layer of both sides, a
// re-paging gather one or more windows.  Runs repage_launch's checks with the destination as the launch's side, and those of
// launch_paged_permute's sources, each side's region at its own page and head count, all before any CUDA call; signals when
// there is nothing to move; then launches kvbm_paged_repage_kernel for a plain re-page, else the gather kernel of the launch's
// unit kind (RepageKernels), and the signal.  max_covered and st: as launch_paged_permute's (st takes the kind's gated kernel, or
// per layer this launch unstreamed).  B: a batch of sequences in place of the one token range (token_begin / token_end unused).
// A routed batch: bit s of a sequence's mask names srcs[s], every mask must be non-zero and below bit num_srcs, and two windows of
// a stage may then share destination heads unless one mask holds both.  Each stage's sources are ANDed with the union of the
// masks, so both gate forms wait on routed sources only, and a CTA has as many warps as the most routed entries of one stage under
// one mask (up to 8).
static cudaError_t launch_paged_repage_gather(const kvbm_stage_source* srcs, int num_srcs, uint32_t src_page, const kvbm_permute_side* dst,
                                              uint32_t dst_num_heads, uint32_t dst_page, uint32_t token_begin, uint32_t token_end,
                                              int layer_begin, int layer_end, uint32_t src_row_bytes, int cast_mode, const float* cast_scales,
                                              uint32_t* done_flag, uint32_t epoch, uint32_t* completion_flag, uint32_t completion_value,
                                              uint32_t max_covered, cudaStream_t stream, const kvbm_permute_stream* st = nullptr,
                                              const RepageBatch* B = nullptr)
{
  RepageLaunch L;
  if (!srcs || num_srcs < 1 || num_srcs > KVBM_GATHER_MAX_SOURCES) return cudaErrorInvalidValue;
  const RepageUnits units = B ? B->kind : kRange;
  const bool route = routed_units(units);
  std::vector<uint32_t> masks;  // a routed batch's distinct source masks
  uint32_t routed = 0;          // and their union
  if (route && B->seqs)
    for (size_t i = 0; i < B->num_seqs; ++i) {
      const uint32_t m = static_cast<const kvbm_route_seq*>(B->seqs)[i].targets;
      if (m == 0 || (m >> num_srcs) != 0) return cudaErrorInvalidValue;
      if (std::find(masks.begin(), masks.end(), m) == masks.end()) masks.push_back(m);
      routed |= m;
    }
  if (!repage_launch(dst, src_page, dst_page, token_begin, token_end, layer_begin, layer_end, src_row_bytes, cast_mode, cast_scales, B, &L))
    return cudaErrorInvalidValue;
  if (L.units == 0) return signal_launch(done_flag, epoch, completion_flag, completion_value, stream);
  const uint32_t nl = L.nl, no = L.no;
  const RowSplit& r = L.r;
  RepageGatherParams P{};
  P.geo = L.geo;
  if (static_cast<uint64_t>(dst_page) * dst_num_heads * L.dst_row_bytes != dst->layout.region_bytes) return cudaErrorInvalidValue;
  if (!fill_permute_side(*dst, nl, no, dst_num_heads, dst_page, static_cast<uint32_t>(L.dst_row_bytes), &P.g.D)) return cudaErrorInvalidValue;
  uint32_t widest;
  if (!fill_stage_sources(srcs, num_srcs, dst_num_heads, nl, no, layer_begin, layer_end, src_page, src_row_bytes, max_covered, &P.g, &widest,
                          route ? &masks : nullptr))
    return cudaErrorInvalidValue;
  P.geo.nh = P.g.covered;
  SourceHeads H{};
  if (route) {
    for (int s = 0; s < num_srcs; ++s) H.n[s] = static_cast<uint16_t>(srcs[s].src.head_count);
    widest = 0;
    for (GatherStage& T : P.g.stage) {
      T.sources &= routed;
      for (uint32_t m : masks) {
        uint32_t n = 0;
        for (int s = 0; s < num_srcs; ++s)
          if ((T.sources & m) >> s & 1u) n += H.n[s];
        widest = std::max(widest, n);
      }
    }
  }
  const int threads = static_cast<int>(std::min<uint32_t>(8, widest)) * 32;
  const unsigned grid = static_cast<unsigned>(L.units);
  if (st)
    return launch_streamed(
        *st, P.g, num_srcs, nl, layer_begin, layer_end, L.units, stream,
        [&](int l) {
          return launch_paged_repage_gather(srcs, num_srcs, src_page, dst, dst_num_heads, dst_page, token_begin, token_end, l, l + 1,
                                            src_row_bytes, cast_mode, cast_scales, nullptr, 0, nullptr, 0, max_covered, stream, nullptr, B);
        },
        [&](const GateArgs& A, unsigned ctas, uint32_t batch) {
          with_repage_units(units, cast_mode, r.pow2, cast_scales != nullptr, L.page_pow2, [&](auto u, auto c, auto p, auto sc, auto pp) {
            const auto kernel = RepageKernels<u>::template gated_gather<c, p, sc, pp>;
            if constexpr (u == kRange)
              kernel<<<ctas, threads, 0, stream>>>(P, A, L.num_big, r, cast_scales, batch);
            else if constexpr (routed_units(u))
              kernel<<<ctas, threads, 0, stream>>>(P, A, H, batch_table<u>(B), L.num_big, r, cast_scales, batch);
            else
              kernel<<<ctas, threads, 0, stream>>>(P, A, batch_table<u>(B), L.num_big, r, cast_scales, batch);
          });
        });
  // a window over every layer and every head of both sides (the checks above make its starts 0)
  const kvbm_permute_source& X = srcs[0].src;
  const bool plain = !B && num_srcs == 1 && whole_layers(srcs[0], nl) && X.head_count == X.num_heads && X.head_count == dst_num_heads;
  RepageParams R{};
  R.big = P.geo.src_small ? P.g.D : P.g.src[0].S;
  R.small = P.geo.src_small ? P.g.src[0].S : P.g.D;
  R.g = P.geo;
  with_repage_units(units, cast_mode, r.pow2, cast_scales != nullptr, L.page_pow2, [&](auto u, auto c, auto p, auto sc, auto pp) {
    const auto kernel = RepageKernels<u>::template gather<c, p, sc, pp>;
    if constexpr (u == kRange) {
      if (plain)
        kvbm_paged_repage_kernel<c, p, sc, pp><<<grid, threads, 0, stream>>>(R, r, cast_scales);
      else
        kernel<<<grid, threads, 0, stream>>>(P, r, cast_scales);
    } else if constexpr (routed_units(u)) {
      kernel<<<grid, threads, 0, stream>>>(P, H, batch_table<u>(B), r, cast_scales);
    } else {
      kernel<<<grid, threads, 0, stream>>>(P, batch_table<u>(B), r, cast_scales);
    }
  });
  return launched(stream, done_flag, epoch, completion_flag, completion_value);
}

// The scatter's target done flags; *any: whether one is set.
static ScatterFlags scatter_flags(const kvbm_scatter_target* targets, int num_targets, bool* any)
{
  ScatterFlags F{};
  *any = false;
  for (int t = 0; t < num_targets; ++t) *any |= (F.done[t] = targets[t].done_flag) != nullptr;
  return F;
}

// The scatter's signal launch: every target's done flag and the completion word, none when all are null.  done_flag (a streamed
// launch's own, nullable) goes with the completion word in a second launch, so that the completion word comes last.
static cudaError_t scatter_signal(const kvbm_scatter_target* targets, int num_targets, uint32_t* done_flag, uint32_t epoch,
                                  uint32_t* completion_flag, uint32_t completion_value, cudaStream_t stream)
{
  bool any;
  const ScatterFlags F = scatter_flags(targets, num_targets, &any);
  uint32_t* last = done_flag ? nullptr : completion_flag;
  if (any || last) {
    kvbm_scatter_signal_kernel<<<1, 1, 0, stream>>>(F, num_targets, epoch, last, completion_value);
    g_launches.fetch_add(1, std::memory_order_relaxed);
    if (const cudaError_t e = cudaGetLastError(); e != cudaSuccess) return e;
  }
  return done_flag ? signal_launch(done_flag, epoch, completion_flag, completion_value, stream) : cudaSuccess;
}

static bool spans_overlap(uint64_t a, uint64_t na, uint64_t b, uint64_t nb) { return a < b + nb && b < a + na; }

// The targets of a scatter from a source of src_nh heads and src_nl layers over source layers [lb, le), into P->tgt, P->stage and
// the entry / pair tables: each target's side (region Pd * its heads * dst_row, the source's outer_dim, its strides over its own
// layers), a non-empty head window and layer window inside both sides, stages whose source layer windows are equal or disjoint
// and tile [lb, le), at most KVBM_GATHER_MAX_HEADS pairs, and no two targets on one pool and table whose destination (layer,
// head) rectangles overlap.  *widest: the most entries of one stage.
static bool fill_scatter_targets(const kvbm_scatter_target* tg, int n, uint32_t src_nh, uint32_t src_nl, uint32_t no, int lb, int le,
                                 uint32_t dst_page, uint64_t dst_row, ScatterParams* P, uint32_t* widest)
{
  int stage_of_tgt[KVBM_GATHER_MAX_SOURCES];
  int num_stages = 0;
  GatherStage* T = P->stage;
  uint32_t pairs = 0;
  for (int t = 0; t < n; ++t) {
    const kvbm_scatter_target& X = tg[t];
    const kvbm_paged_layout& L = X.side.layout;
    if (!X.side.block_ids || !L.layer_base || L.outer_dim != no) return false;
    if (static_cast<uint64_t>(dst_page) * X.num_heads * dst_row != L.region_bytes) return false;
    if (!fill_permute_side(X.side, L.num_layers, no, X.num_heads, dst_page, static_cast<uint32_t>(dst_row), &P->tgt[t].D)) return false;
    if (X.head_count == 0 || static_cast<uint64_t>(X.src_head_begin) + X.head_count > src_nh ||
        static_cast<uint64_t>(X.dst_head_begin) + X.head_count > X.num_heads)
      return false;
    const uint64_t src_end = static_cast<uint64_t>(X.src_layer_begin) + X.layer_count;
    if (X.layer_count == 0 || src_end > src_nl || static_cast<uint64_t>(X.dst_layer_begin) + X.layer_count > L.num_layers) return false;
    if ((pairs += X.head_count) > KVBM_GATHER_MAX_HEADS) return false;
    const int k = stage_of_tgt[t] = window_stage(T, &num_stages, X.src_layer_begin, static_cast<uint32_t>(src_end));
    if (k < 0) return false;
    T[k].sources = 1;  // the one source
    for (int u = 0; u < t; ++u) {
      const kvbm_scatter_target& Y = tg[u];
      if (Y.side.layout.layer_base == L.layer_base && Y.side.block_ids == X.side.block_ids &&
          spans_overlap(X.dst_layer_begin, X.layer_count, Y.dst_layer_begin, Y.layer_count) &&
          spans_overlap(X.dst_head_begin, X.head_count, Y.dst_head_begin, Y.head_count))
        return false;
    }
    P->tgt[t].shift = X.dst_layer_begin - X.src_layer_begin;
    P->tgt[t].head_delta = X.dst_head_begin - X.src_head_begin;
  }
  int order[KVBM_GATHER_MAX_SOURCES];
  if (!order_stages(T, num_stages, lb, le, order)) return false;
  // per stage: its (source head, target) pairs in ascending head, then target order, one entry per head
  GatherStage sorted[KVBM_GATHER_MAX_SOURCES] = {};
  uint32_t entries = 0, p = 0;
  *widest = 0;
  for (int i = 0; i < num_stages; ++i) {
    GatherStage& S = sorted[i] = T[order[i]];
    S.first = entries;
    uint32_t hs[KVBM_GATHER_MAX_HEADS];
    uint8_t ts[KVBM_GATHER_MAX_HEADS];
    uint32_t m = 0;
    for (int t = 0; t < n; ++t) {
      if (stage_of_tgt[t] != order[i]) continue;
      for (uint32_t h = tg[t].src_head_begin; h < tg[t].src_head_begin + tg[t].head_count; ++h) {
        uint32_t at = m++;
        while (at > 0 && hs[at - 1] > h) {  // stable: a head's pairs stay in target order
          hs[at] = hs[at - 1];
          ts[at] = ts[at - 1];
          --at;
        }
        hs[at] = h;
        ts[at] = static_cast<uint8_t>(t);
      }
    }
    for (uint32_t a = 0; a < m; ++a, ++p) {
      if (a == 0 || hs[a] != hs[a - 1]) {
        P->head[entries] = hs[a];
        P->pair_first[entries++] = static_cast<uint16_t>(p);
      }
      P->pair_tgt[p] = ts[a];
    }
    S.count = entries - S.first;
    *widest = std::max(*widest, S.count);
  }
  P->pair_first[entries] = static_cast<uint16_t>(p);
  std::copy(sorted, sorted + KVBM_GATHER_MAX_SOURCES, T);
  return true;
}

// The scatter: every check before any CUDA call (repage_launch's with the source as the launch's side, and the target-count rule
// before them), then one kvbm_paged_repage_scatter_kernel launch and the signal.  st: a streamed launch (its flags are the ones
// passed, and its done flag is written with the targets'), which takes the gated push kernel, or per source layer this launch
// unstreamed.  B: a batch of sequences in place of the one token range (token_begin / token_end unused), which takes its kind's
// kernels (RepageKernels); a routed batch's every target mask must be non-zero and below bit num_targets.
static cudaError_t launch_paged_repage_scatter(const kvbm_permute_side* src, uint32_t src_num_heads, uint32_t src_page,
                                               const kvbm_scatter_target* targets, int num_targets, uint32_t dst_page, uint32_t token_begin,
                                               uint32_t token_end, int layer_begin, int layer_end, uint32_t src_row_bytes, int cast_mode,
                                               const float* cast_scales, uint32_t epoch, uint32_t* completion_flag, uint32_t completion_value,
                                               cudaStream_t stream, const kvbm_permute_stream* st = nullptr, const RepageBatch* B = nullptr)
{
  RepageLaunch L;
  if (!targets || num_targets < 1 || num_targets > KVBM_GATHER_MAX_SOURCES) return cudaErrorInvalidValue;
  const RepageUnits units = B ? B->kind : kRange;
  if (routed_units(units) && B->seqs)
    for (size_t i = 0; i < B->num_seqs; ++i) {
      const uint32_t m = static_cast<const kvbm_route_seq*>(B->seqs)[i].targets;
      if (m == 0 || (m >> num_targets) != 0) return cudaErrorInvalidValue;
    }
  if (!repage_launch(src, src_page, dst_page, token_begin, token_end, layer_begin, layer_end, src_row_bytes, cast_mode, cast_scales, B, &L))
    return cudaErrorInvalidValue;
  if (L.units == 0) return scatter_signal(targets, num_targets, st ? st->done_flag : nullptr, epoch, completion_flag, completion_value, stream);
  const uint32_t nl = L.nl, no = L.no;
  const RowSplit& r = L.r;
  ScatterParams P{};
  P.geo = L.geo;
  if (static_cast<uint64_t>(src_page) * src_num_heads * src_row_bytes != src->layout.region_bytes) return cudaErrorInvalidValue;
  if (!fill_permute_side(*src, nl, no, src_num_heads, src_page, src_row_bytes, &P.S)) return cudaErrorInvalidValue;
  uint32_t widest;
  if (!fill_scatter_targets(targets, num_targets, src_num_heads, nl, no, layer_begin, layer_end, dst_page, L.dst_row_bytes, &P, &widest))
    return cudaErrorInvalidValue;
  const int threads = static_cast<int>(std::min<uint32_t>(8, widest)) * 32;
  if (st) {
    // the stream-wait form writes the targets' done flags after the last layer only
    kvbm_scatter_target quiet[KVBM_GATHER_MAX_SOURCES];
    std::copy(targets, targets + num_targets, quiet);
    for (int t = 0; t < num_targets; ++t) quiet[t].done_flag = nullptr;
    return launch_streamed(
        *st, P, 1, nl, layer_begin, layer_end, L.units, stream,
        [&](int l) {
          return launch_paged_repage_scatter(src, src_num_heads, src_page, l + 1 == layer_end ? targets : quiet, num_targets, dst_page,
                                             token_begin, token_end, l, l + 1, src_row_bytes, cast_mode, cast_scales, epoch, nullptr, 0,
                                             stream, nullptr, B);
        },
        [&](const GateArgs& A, unsigned ctas, uint32_t batch) {
          GateArgs Ag = A;
          bool any;
          const ScatterFlags F = scatter_flags(targets, num_targets, &any);
          Ag.ss.want_done |= any;
          with_repage_units(units, cast_mode, r.pow2, cast_scales != nullptr, L.page_pow2, [&](auto u, auto c, auto p, auto sc, auto pp) {
            const auto kernel = RepageKernels<u>::template gated_scatter<c, p, sc, pp>;
            if constexpr (u == kRange)
              kernel<<<ctas, threads, 0, stream>>>(P, Ag, F, num_targets, L.num_big, r, cast_scales, batch);
            else
              kernel<<<ctas, threads, 0, stream>>>(P, Ag, F, num_targets, batch_table<u>(B), L.num_big, r, cast_scales, batch);
          });
        });
  }
  const unsigned grid = static_cast<unsigned>(L.units);
  with_repage_units(units, cast_mode, r.pow2, cast_scales != nullptr, L.page_pow2, [&](auto u, auto c, auto p, auto sc, auto pp) {
    const auto kernel = RepageKernels<u>::template scatter<c, p, sc, pp>;
    if constexpr (u == kRange)
      kernel<<<grid, threads, 0, stream>>>(P, r, cast_scales);
    else
      kernel<<<grid, threads, 0, stream>>>(P, batch_table<u>(B), r, cast_scales);
  });
  g_launches.fetch_add(1, std::memory_order_relaxed);
  const cudaError_t e = cudaGetLastError();
  return e != cudaSuccess ? e : scatter_signal(targets, num_targets, nullptr, epoch, completion_flag, completion_value, stream);
}

}  // namespace kvbm

using namespace kvbm;

// =================================================================================================
// C ABI -- Part 1 (reference symbols)
// =================================================================================================
extern "C" cudaError_t
kvbm_kernels_launch_vectorized_copy(void** src_ptrs, void** dst_ptrs, size_t copy_size_bytes, int num_pairs,
                                    cudaStream_t stream)
{
  if (num_pairs == 0 || copy_size_bytes == 0) return cudaSuccess;  // tensor_kernels.cu:555-557
  if (!src_ptrs || !dst_ptrs) return cudaErrorInvalidValue;        // :559-561
  if (num_pairs < 0) return cudaErrorInvalidValue;
  DeviceInfo di;
  cudaError_t e = device_info(&di);
  if (e != cudaSuccess) return e;

  const uint64_t pairs = static_cast<uint64_t>(num_pairs);
  uint64_t ctas;
  uint32_t chunks_per_pair = 1;
  if (copy_size_bytes <= kPairSmall) {
    ctas = (pairs + kPairThreads / 32 - 1) / (kPairThreads / 32);  // one warp per pair
  } else {
    const uint64_t cpp = (copy_size_bytes + kPairChunk - 1) / kPairChunk;
    if (cpp >= (1ull << 32)) return cudaErrorInvalidValue;
    chunks_per_pair = static_cast<uint32_t>(cpp);
    ctas = pairs * cpp;
  }
  const uint64_t gx = std::min<uint64_t>(ctas, 1ull << 30);
  const uint64_t gy = (ctas + gx - 1) / gx;
  if (gy > 65535) return cudaErrorInvalidValue;
  kvbm_pair_copy_kernel<<<dim3(static_cast<unsigned>(gx), static_cast<unsigned>(gy)), kPairThreads, 0, stream>>>(
      src_ptrs, dst_ptrs, copy_size_bytes, chunks_per_pair, pairs);
  g_launches.fetch_add(1, std::memory_order_relaxed);
  return cudaGetLastError();  // :570
}

extern "C" cudaError_t
kvbm_kernels_memcpy_batch(const void* const* src_ptrs, void* const* dst_ptrs, size_t size_per_copy,
                          size_t num_copies, int mode, cudaStream_t stream)
{
  if (num_copies == 0 || size_per_copy == 0) return cudaSuccess;  // tensor_kernels.cu:396-398
  if (!src_ptrs || !dst_ptrs) return cudaErrorInvalidValue;       // :400-402

  auto one_by_one = [&]() -> cudaError_t {
    for (size_t i = 0; i < num_copies; ++i) {
      cudaError_t e = cudaMemcpyAsync(dst_ptrs[i], src_ptrs[i], size_per_copy, cudaMemcpyDefault, stream);
      if (e != cudaSuccess) return e;
    }
    return cudaSuccess;
  };
  if (mode == KVBM_MEMCPY_FALLBACK_ONLY) return one_by_one();

#if CUDART_VERSION >= 12090
  // Host tables are consumed before returning (the caller may free them immediately: cuda.rs:185-204).
  std::vector<void*> srcs(num_copies), dsts(num_copies);
  std::vector<size_t> sizes(num_copies, size_per_copy), attr_idx(num_copies, 0);
  for (size_t i = 0; i < num_copies; ++i) {
    srcs[i] = const_cast<void*>(src_ptrs[i]);
    dsts[i] = dst_ptrs[i];
  }
  cudaMemcpyAttributes attr = {};
  attr.srcAccessOrder = cudaMemcpySrcAccessOrderStream;
#if CUDART_VERSION >= 13000
  cudaError_t e = cudaMemcpyBatchAsync(dsts.data(), srcs.data(), sizes.data(), num_copies, &attr, attr_idx.data(), 1, stream);
#else
  size_t fail_idx = 0;
  cudaError_t e = cudaMemcpyBatchAsync(dsts.data(), srcs.data(), sizes.data(), num_copies, &attr, attr_idx.data(), 1,
                                       &fail_idx, stream);
#endif
  if (e == cudaErrorNotSupported || e == cudaErrorInvalidValue) {
    if (mode == KVBM_MEMCPY_BATCH_WITHOUT_FALLBACK) return e;
    (void)cudaGetLastError();
    return one_by_one();
  }
  return e;
#else
  if (mode == KVBM_MEMCPY_BATCH_WITHOUT_FALLBACK) return cudaErrorNotSupported;
  return one_by_one();
#endif
}

extern "C" cudaError_t
kvbm_kernels_launch_universal_from_block(void* const* universal_ptrs, const void* const* block_ptrs,
                                         size_t num_blocks, size_t nh, size_t nl, size_t no, size_t nt, size_t hd,
                                         int dtype, int layout, cudaStream_t stream)
{
  return launch_permute<true>(universal_ptrs, const_cast<void* const*>(reinterpret_cast<const void* const*>(block_ptrs)),
                              num_blocks, nh, nl, no, nt, hd, dtype, layout, stream);
}

extern "C" cudaError_t
kvbm_kernels_launch_block_from_universal(const void* const* universal_ptrs, void* const* block_ptrs,
                                         size_t num_blocks, size_t nh, size_t nl, size_t no, size_t nt, size_t hd,
                                         int dtype, int layout, cudaStream_t stream)
{
  return launch_permute<false>(const_cast<void* const*>(reinterpret_cast<const void* const*>(universal_ptrs)), block_ptrs,
                               num_blocks, nh, nl, no, nt, hd, dtype, layout, stream);
}

// Host-only view of the stride table the permuting kernel walks with (no GPU needed): lets the CPU suite check the
// address arithmetic of every KvBlockLayout against the oracle's dim_order definition, at sizes no GPU test allocates.
extern "C" int
kvbm_kernels_permute_strides(int kv_layout, uint32_t num_layers, uint32_t outer_dim, uint32_t num_heads, uint32_t page_size,
                             uint32_t row_bytes, uint64_t block_stride, uint64_t outer_stride, uint64_t out[5])
{
  if (!out) return 1;
  kvbm_permute_side side{};
  side.layout.block_stride = block_stride;
  side.layout.outer_stride = outer_stride;
  side.kv_layout = kv_layout;
  PermuteSide p;
  if (!fill_permute_side(side, num_layers, outer_dim, num_heads, page_size, row_bytes, &p)) return 1;
  out[0] = p.universal ? 1 : 0;  // 1: offsets are relative to the block's start; 0: relative to the (layer, outer) region
  out[1] = p.layer_step;
  out[2] = p.outer_step;
  out[3] = p.head_stride;
  out[4] = p.tok_stride;
  return 0;
}

extern "C" cudaError_t
kvbm_kernels_paged_permute(const kvbm_permute_side* src, const kvbm_permute_side* dst, int num_blocks, int layer_begin,
                           int layer_end, uint32_t num_heads, uint32_t page_size, uint32_t row_bytes, uint32_t* done_flag,
                           uint32_t epoch, uint32_t* completion_flag, uint32_t completion_value, cudaStream_t stream)
{
  return kvbm_kernels_paged_permute_cast(src, dst, num_blocks, layer_begin, layer_end, num_heads, page_size, row_bytes, KVBM_CAST_NONE,
                                         done_flag, epoch, completion_flag, completion_value, stream);
}

extern "C" cudaError_t
kvbm_kernels_paged_permute_cast(const kvbm_permute_side* src, const kvbm_permute_side* dst, int num_blocks, int layer_begin,
                                int layer_end, uint32_t num_heads, uint32_t page_size, uint32_t src_row_bytes, int cast_mode,
                                uint32_t* done_flag, uint32_t epoch, uint32_t* completion_flag, uint32_t completion_value,
                                cudaStream_t stream)
{
  return kvbm_kernels_paged_permute_heads(src, dst, num_blocks, layer_begin, layer_end, num_heads, 0, num_heads, 0, num_heads, page_size,
                                          src_row_bytes, cast_mode, done_flag, epoch, completion_flag, completion_value, stream);
}

extern "C" cudaError_t
kvbm_kernels_paged_permute_heads(const kvbm_permute_side* src, const kvbm_permute_side* dst, int num_blocks, int layer_begin,
                                 int layer_end, uint32_t src_num_heads, uint32_t src_head_begin, uint32_t dst_num_heads,
                                 uint32_t dst_head_begin, uint32_t head_count, uint32_t page_size, uint32_t src_row_bytes, int cast_mode,
                                 uint32_t* done_flag, uint32_t epoch, uint32_t* completion_flag, uint32_t completion_value,
                                 cudaStream_t stream)
{
  return kvbm_kernels_paged_permute_heads_scaled(src, dst, num_blocks, layer_begin, layer_end, src_num_heads, src_head_begin, dst_num_heads,
                                                 dst_head_begin, head_count, page_size, src_row_bytes, cast_mode, nullptr, done_flag, epoch,
                                                 completion_flag, completion_value, stream);
}

extern "C" cudaError_t
kvbm_kernels_paged_permute_heads_scaled(const kvbm_permute_side* src, const kvbm_permute_side* dst, int num_blocks, int layer_begin,
                                        int layer_end, uint32_t src_num_heads, uint32_t src_head_begin, uint32_t dst_num_heads,
                                        uint32_t dst_head_begin, uint32_t head_count, uint32_t page_size, uint32_t src_row_bytes,
                                        int cast_mode, const float* cast_scales, uint32_t* done_flag, uint32_t epoch,
                                        uint32_t* completion_flag, uint32_t completion_value, cudaStream_t stream)
{
  const kvbm_permute_source one{src ? *src : kvbm_permute_side{}, src_num_heads, src_head_begin, dst_head_begin, head_count};
  kvbm_stage_source staged[1];
  return launch_paged_permute(one_stage(&one, 1, dst, staged), 1, dst, dst_num_heads, num_blocks, layer_begin, layer_end, page_size,
                              src_row_bytes, cast_mode, cast_scales, done_flag, epoch, completion_flag, completion_value, UINT32_MAX, stream);
}

extern "C" cudaError_t
kvbm_kernels_paged_permute_gather(const kvbm_permute_source* srcs, int num_srcs, const kvbm_permute_side* dst, uint32_t dst_num_heads,
                                  int num_blocks, int layer_begin, int layer_end, uint32_t page_size, uint32_t src_row_bytes,
                                  int cast_mode, uint32_t* done_flag, uint32_t epoch, uint32_t* completion_flag,
                                  uint32_t completion_value, cudaStream_t stream)
{
  return kvbm_kernels_paged_permute_gather_scaled(srcs, num_srcs, dst, dst_num_heads, num_blocks, layer_begin, layer_end, page_size,
                                                  src_row_bytes, cast_mode, nullptr, done_flag, epoch, completion_flag, completion_value,
                                                  stream);
}

extern "C" cudaError_t
kvbm_kernels_paged_permute_gather_scaled(const kvbm_permute_source* srcs, int num_srcs, const kvbm_permute_side* dst,
                                         uint32_t dst_num_heads, int num_blocks, int layer_begin, int layer_end, uint32_t page_size,
                                         uint32_t src_row_bytes, int cast_mode, const float* cast_scales, uint32_t* done_flag,
                                         uint32_t epoch, uint32_t* completion_flag, uint32_t completion_value, cudaStream_t stream)
{
  kvbm_stage_source staged[KVBM_GATHER_MAX_SOURCES];
  return launch_paged_permute(one_stage(srcs, num_srcs, dst, staged), num_srcs, dst, dst_num_heads, num_blocks, layer_begin, layer_end,
                              page_size, src_row_bytes, cast_mode, cast_scales, done_flag, epoch, completion_flag, completion_value,
                              KVBM_GATHER_MAX_HEADS, stream);
}

extern "C" cudaError_t
kvbm_kernels_paged_repage(const kvbm_permute_side* src, uint32_t src_page_size, const kvbm_permute_side* dst, uint32_t dst_page_size,
                          uint32_t token_begin, uint32_t token_end, int layer_begin, int layer_end, uint32_t num_heads,
                          uint32_t src_row_bytes, int cast_mode, const float* cast_scales, uint32_t* done_flag, uint32_t epoch,
                          uint32_t* completion_flag, uint32_t completion_value, cudaStream_t stream)
{
  const kvbm_permute_source one{src ? *src : kvbm_permute_side{}, num_heads, 0, 0, num_heads};
  kvbm_stage_source staged[1];
  return launch_paged_repage_gather(one_stage(&one, 1, dst, staged), 1, src_page_size, dst, num_heads, dst_page_size, token_begin, token_end,
                                    layer_begin, layer_end, src_row_bytes, cast_mode, cast_scales, done_flag, epoch, completion_flag,
                                    completion_value, UINT32_MAX, stream);
}

extern "C" cudaError_t
kvbm_kernels_paged_repage_gather(const kvbm_permute_source* srcs, int num_srcs, uint32_t src_page_size, const kvbm_permute_side* dst,
                                 uint32_t dst_num_heads, uint32_t dst_page_size, uint32_t token_begin, uint32_t token_end, int layer_begin,
                                 int layer_end, uint32_t src_row_bytes, int cast_mode, const float* cast_scales, uint32_t* done_flag,
                                 uint32_t epoch, uint32_t* completion_flag, uint32_t completion_value, cudaStream_t stream)
{
  kvbm_stage_source staged[KVBM_GATHER_MAX_SOURCES];
  return launch_paged_repage_gather(one_stage(srcs, num_srcs, dst, staged), num_srcs, src_page_size, dst, dst_num_heads, dst_page_size,
                                    token_begin, token_end, layer_begin, layer_end, src_row_bytes, cast_mode, cast_scales, done_flag, epoch,
                                    completion_flag, completion_value, KVBM_GATHER_MAX_HEADS, stream);
}

extern "C" cudaError_t
kvbm_kernels_paged_permute_gather_streamed(const kvbm_permute_source* srcs, int num_srcs, const kvbm_permute_side* dst, uint32_t dst_num_heads,
                                           int num_blocks, int layer_begin, int layer_end, uint32_t page_size, uint32_t src_row_bytes,
                                           int cast_mode, const float* cast_scales, const kvbm_permute_stream* st, cudaStream_t stream)
{
  if (!stream_args_ok(st, num_srcs)) return cudaErrorInvalidValue;
  kvbm_stage_source staged[KVBM_GATHER_MAX_SOURCES];
  return launch_paged_permute(one_stage(srcs, num_srcs, dst, staged), num_srcs, dst, dst_num_heads, num_blocks, layer_begin, layer_end,
                              page_size, src_row_bytes, cast_mode, cast_scales, st->done_flag, st->epoch, st->completion_flag,
                              st->completion_value, KVBM_GATHER_MAX_HEADS, stream, st);
}

extern "C" cudaError_t
kvbm_kernels_paged_stage_repage_gather(const kvbm_stage_source* srcs, int num_srcs, uint32_t src_page_size, const kvbm_permute_side* dst,
                                       uint32_t dst_num_heads, uint32_t dst_page_size, uint32_t token_begin, uint32_t token_end,
                                       int layer_begin, int layer_end, uint32_t src_row_bytes, int cast_mode, const float* cast_scales,
                                       uint32_t* done_flag, uint32_t epoch, uint32_t* completion_flag, uint32_t completion_value,
                                       cudaStream_t stream)
{
  return launch_paged_repage_gather(srcs, num_srcs, src_page_size, dst, dst_num_heads, dst_page_size, token_begin, token_end, layer_begin,
                                    layer_end, src_row_bytes, cast_mode, cast_scales, done_flag, epoch, completion_flag, completion_value,
                                    KVBM_GATHER_MAX_HEADS, stream);
}

extern "C" cudaError_t
kvbm_kernels_paged_stage_repage_gather_streamed(const kvbm_stage_source* srcs, int num_srcs, uint32_t src_page_size,
                                                const kvbm_permute_side* dst, uint32_t dst_num_heads, uint32_t dst_page_size,
                                                uint32_t token_begin, uint32_t token_end, int layer_begin, int layer_end,
                                                uint32_t src_row_bytes, int cast_mode, const float* cast_scales,
                                                const kvbm_permute_stream* st, cudaStream_t stream)
{
  if (!stream_args_ok(st, num_srcs)) return cudaErrorInvalidValue;
  return launch_paged_repage_gather(srcs, num_srcs, src_page_size, dst, dst_num_heads, dst_page_size, token_begin, token_end, layer_begin,
                                    layer_end, src_row_bytes, cast_mode, cast_scales, st->done_flag, st->epoch, st->completion_flag,
                                    st->completion_value, KVBM_GATHER_MAX_HEADS, stream, st);
}

// kvbm_kernels_repage_batch_units over ranges of either sequence type; the fourth word of each unit is last(i, phase) of its
// sequence i and the block's phase (0 unless `any`).  any: pages that need not divide (kvbm_kernels_repage_anypage_units).
template <class Seq, class Unit, class Last>
static int batch_units(const Seq* seqs, size_t num_seqs, uint32_t src_page_size, uint32_t dst_page_size, Unit* out, size_t cap,
                       size_t* num_units, size_t* src_ids, size_t* dst_ids, Last last, bool any = false)
{
  if ((num_seqs && !seqs) || (cap && !out) || !num_units || !src_ids || !dst_ids) return 1;
  if (src_page_size == 0 || dst_page_size == 0) return 1;
  const bool src_small = src_page_size < dst_page_size;
  const uint64_t big = src_small ? dst_page_size : src_page_size, small = src_small ? src_page_size : dst_page_size;
  if ((!any && big % small) || !repage_exact(big, small)) return 1;
  for (size_t i = 0; i < num_seqs; ++i) {
    if (seqs[i].token_end < seqs[i].token_begin) return 1;
    if (seqs[i].token_end != seqs[i].token_begin && (seqs[i].token_end + big - 1) / big * big >= (1ull << 32)) return 1;
  }
  size_t nb = 0, ns = 0;
  for (size_t i = 0; i < num_seqs; ++i) {
    const uint64_t tb = seqs[i].token_begin, te = seqs[i].token_end;
    if (tb == te) continue;
    const uint64_t big_first = tb / big, big_end = (te + big - 1) / big, small_first = tb / small, small_end = (te + small - 1) / small;
    uint64_t j = big_first;
    for (; j < big_end && nb < cap; ++j, ++nb) {
      const uint64_t first = j * big, t0 = std::max(tb, first), t1 = std::min(te, first + big);
      // the concatenated small table's entry of the small block that holds the block's slot 0 (j * ratio with dividing pages): below
      // 0 (wrapping) when it lies before the range; the phase is that slot 0's slot in it
      out[nb] = Unit{static_cast<uint32_t>(t0 - first), static_cast<uint32_t>(t1 - t0), static_cast<uint32_t>(ns + first / small - small_first),
                     last(i, static_cast<uint32_t>(first % small))};
    }
    nb += static_cast<size_t>(big_end - j);  // past the capacity: counted, not written
    ns += static_cast<size_t>(small_end - small_first);
  }
  *num_units = nb;
  *src_ids = src_small ? ns : nb;
  *dst_ids = src_small ? nb : ns;
  return 0;
}

extern "C" int
kvbm_kernels_repage_batch_units(const kvbm_repage_seq* seqs, size_t num_seqs, uint32_t src_page_size, uint32_t dst_page_size,
                                kvbm_repage_unit* out, size_t cap, size_t* num_units, size_t* src_ids, size_t* dst_ids)
{
  return batch_units(seqs, num_seqs, src_page_size, dst_page_size, out, cap, num_units, src_ids, dst_ids,
                     [](size_t i, uint32_t) { return static_cast<uint32_t>(i); });
}

extern "C" int
kvbm_kernels_repage_route_units(const kvbm_route_seq* seqs, size_t num_seqs, uint32_t src_page_size, uint32_t dst_page_size,
                                kvbm_route_unit* out, size_t cap, size_t* num_units, size_t* src_ids, size_t* dst_ids)
{
  return batch_units(seqs, num_seqs, src_page_size, dst_page_size, out, cap, num_units, src_ids, dst_ids,
                     [seqs](size_t i, uint32_t) { return seqs[i].targets; });
}

extern "C" int
kvbm_kernels_repage_anypage_units(const kvbm_repage_seq* seqs, size_t num_seqs, uint32_t src_page_size, uint32_t dst_page_size,
                                  kvbm_repage_anypage_unit* out, size_t cap, size_t* num_units, size_t* src_ids, size_t* dst_ids)
{
  return batch_units(seqs, num_seqs, src_page_size, dst_page_size, out, cap, num_units, src_ids, dst_ids,
                     [](size_t, uint32_t phase) { return phase; }, /*any=*/true);
}

extern "C" int
kvbm_kernels_repage_route_anypage_units(const kvbm_route_seq* seqs, size_t num_seqs, uint32_t src_page_size, uint32_t dst_page_size,
                                        kvbm_route_anypage_unit* out, size_t cap, size_t* num_units, size_t* src_ids, size_t* dst_ids)
{
  // the mask takes the low half of the fourth word; the phase, below a small page the exactness bound keeps under 2^16, the high
  for (size_t i = 0; seqs && i < num_seqs; ++i)
    if (seqs[i].targets >> 16) return 1;
  return batch_units(seqs, num_seqs, src_page_size, dst_page_size, out, cap, num_units, src_ids, dst_ids,
                     [seqs](size_t i, uint32_t phase) { return seqs[i].targets | phase << 16; }, /*any=*/true);
}

// The body of every batch re-paging gather entry: a batch of UNITS, streamed through st (checked here, and then with st's flags),
// else with the flags passed.  A streamed routed batch needs the ready flags of the sources some sequence is routed to only.
template <RepageUnits UNITS>
static cudaError_t repage_gather_batch(const kvbm_stage_source* srcs, int num_srcs, uint32_t src_page_size, const kvbm_permute_side* dst,
                                       uint32_t dst_num_heads, uint32_t dst_page_size, const typename RepageKernels<UNITS>::Seq* seqs,
                                       size_t num_seqs, const typename RepageKernels<UNITS>::Record* units, size_t num_units, int layer_begin,
                                       int layer_end, uint32_t src_row_bytes, int cast_mode, const float* cast_scales, bool streamed,
                                       const kvbm_permute_stream* st, uint32_t* done_flag, uint32_t epoch, uint32_t* completion_flag,
                                       uint32_t completion_value, cudaStream_t stream)
{
  if (streamed) {
    uint32_t used = ~0u;
    if constexpr (routed_units(UNITS)) {
      used = 0;
      for (size_t i = 0; seqs && i < num_seqs; ++i) used |= seqs[i].targets;
    }
    if (!stream_args_ok(st, num_srcs, used)) return cudaErrorInvalidValue;
    done_flag = st->done_flag;
    epoch = st->epoch;
    completion_flag = st->completion_flag;
    completion_value = st->completion_value;
  }
  const RepageBatch B = repage_batch<UNITS>(seqs, num_seqs, units, num_units);
  return launch_paged_repage_gather(srcs, num_srcs, src_page_size, dst, dst_num_heads, dst_page_size, 0, 0, layer_begin, layer_end,
                                    src_row_bytes, cast_mode, cast_scales, done_flag, epoch, completion_flag, completion_value,
                                    KVBM_GATHER_MAX_HEADS, stream, st, &B);
}

// The body of every batch scatter entry: a batch of UNITS, streamed through st (checked here, and then with st's flags), else
// with the flags passed.
template <RepageUnits UNITS>
static cudaError_t repage_scatter_batch(const kvbm_permute_side* src, uint32_t src_num_heads, uint32_t src_page_size,
                                        const kvbm_scatter_target* targets, int num_targets, uint32_t dst_page_size,
                                        const typename RepageKernels<UNITS>::Seq* seqs, size_t num_seqs,
                                        const typename RepageKernels<UNITS>::Record* units, size_t num_units, int layer_begin, int layer_end,
                                        uint32_t src_row_bytes, int cast_mode, const float* cast_scales, bool streamed,
                                        const kvbm_permute_stream* st, uint32_t epoch, uint32_t* completion_flag, uint32_t completion_value,
                                        cudaStream_t stream)
{
  if (streamed) {
    if (!stream_args_ok(st, 1)) return cudaErrorInvalidValue;
    epoch = st->epoch;
    completion_flag = st->completion_flag;
    completion_value = st->completion_value;
  }
  const RepageBatch B = repage_batch<UNITS>(seqs, num_seqs, units, num_units);
  return launch_paged_repage_scatter(src, src_num_heads, src_page_size, targets, num_targets, dst_page_size, 0, 0, layer_begin, layer_end,
                                     src_row_bytes, cast_mode, cast_scales, epoch, completion_flag, completion_value, stream, st, &B);
}

extern "C" cudaError_t
kvbm_kernels_paged_stage_repage_gather_anypage(const kvbm_stage_source* srcs, int num_srcs, uint32_t src_page_size, const kvbm_permute_side* dst,
                                               uint32_t dst_num_heads, uint32_t dst_page_size, const kvbm_repage_seq* seqs, size_t num_seqs,
                                               const kvbm_repage_anypage_unit* units, size_t num_units, int layer_begin, int layer_end,
                                               uint32_t src_row_bytes, int cast_mode, const float* cast_scales, uint32_t* done_flag,
                                               uint32_t epoch, uint32_t* completion_flag, uint32_t completion_value, cudaStream_t stream)
{
  return repage_gather_batch<kPhased>(srcs, num_srcs, src_page_size, dst, dst_num_heads, dst_page_size, seqs, num_seqs, units, num_units,
                                      layer_begin, layer_end, src_row_bytes, cast_mode, cast_scales, false, nullptr, done_flag, epoch,
                                      completion_flag, completion_value, stream);
}

extern "C" cudaError_t
kvbm_kernels_paged_stage_repage_gather_anypage_streamed(const kvbm_stage_source* srcs, int num_srcs, uint32_t src_page_size,
                                                        const kvbm_permute_side* dst, uint32_t dst_num_heads, uint32_t dst_page_size,
                                                        const kvbm_repage_seq* seqs, size_t num_seqs, const kvbm_repage_anypage_unit* units,
                                                        size_t num_units, int layer_begin, int layer_end, uint32_t src_row_bytes,
                                                        int cast_mode, const float* cast_scales, const kvbm_permute_stream* st,
                                                        cudaStream_t stream)
{
  return repage_gather_batch<kPhased>(srcs, num_srcs, src_page_size, dst, dst_num_heads, dst_page_size, seqs, num_seqs, units, num_units,
                                      layer_begin, layer_end, src_row_bytes, cast_mode, cast_scales, true, st, nullptr, 0, nullptr, 0,
                                      stream);
}

extern "C" cudaError_t
kvbm_kernels_paged_stage_repage_gather_batch(const kvbm_stage_source* srcs, int num_srcs, uint32_t src_page_size, const kvbm_permute_side* dst,
                                             uint32_t dst_num_heads, uint32_t dst_page_size, const kvbm_repage_seq* seqs, size_t num_seqs,
                                             const kvbm_repage_unit* units, size_t num_units, int layer_begin, int layer_end,
                                             uint32_t src_row_bytes, int cast_mode, const float* cast_scales, uint32_t* done_flag,
                                             uint32_t epoch, uint32_t* completion_flag, uint32_t completion_value, cudaStream_t stream)
{
  return repage_gather_batch<kSeqs>(srcs, num_srcs, src_page_size, dst, dst_num_heads, dst_page_size, seqs, num_seqs, units, num_units,
                                    layer_begin, layer_end, src_row_bytes, cast_mode, cast_scales, false, nullptr, done_flag, epoch,
                                    completion_flag, completion_value, stream);
}

extern "C" cudaError_t
kvbm_kernels_paged_stage_repage_gather_batch_streamed(const kvbm_stage_source* srcs, int num_srcs, uint32_t src_page_size,
                                                      const kvbm_permute_side* dst, uint32_t dst_num_heads, uint32_t dst_page_size,
                                                      const kvbm_repage_seq* seqs, size_t num_seqs, const kvbm_repage_unit* units,
                                                      size_t num_units, int layer_begin, int layer_end, uint32_t src_row_bytes,
                                                      int cast_mode, const float* cast_scales, const kvbm_permute_stream* st,
                                                      cudaStream_t stream)
{
  return repage_gather_batch<kSeqs>(srcs, num_srcs, src_page_size, dst, dst_num_heads, dst_page_size, seqs, num_seqs, units, num_units,
                                    layer_begin, layer_end, src_row_bytes, cast_mode, cast_scales, true, st, nullptr, 0, nullptr, 0,
                                    stream);
}

extern "C" cudaError_t
kvbm_kernels_paged_stage_repage_gather_routed(const kvbm_stage_source* srcs, int num_srcs, uint32_t src_page_size, const kvbm_permute_side* dst,
                                              uint32_t dst_num_heads, uint32_t dst_page_size, const kvbm_route_seq* seqs, size_t num_seqs,
                                              const kvbm_route_unit* units, size_t num_units, int layer_begin, int layer_end,
                                              uint32_t src_row_bytes, int cast_mode, const float* cast_scales, uint32_t* done_flag,
                                              uint32_t epoch, uint32_t* completion_flag, uint32_t completion_value, cudaStream_t stream)
{
  return repage_gather_batch<kRouted>(srcs, num_srcs, src_page_size, dst, dst_num_heads, dst_page_size, seqs, num_seqs, units, num_units,
                                      layer_begin, layer_end, src_row_bytes, cast_mode, cast_scales, false, nullptr, done_flag, epoch,
                                      completion_flag, completion_value, stream);
}

extern "C" cudaError_t
kvbm_kernels_paged_stage_repage_gather_routed_streamed(const kvbm_stage_source* srcs, int num_srcs, uint32_t src_page_size,
                                                       const kvbm_permute_side* dst, uint32_t dst_num_heads, uint32_t dst_page_size,
                                                       const kvbm_route_seq* seqs, size_t num_seqs, const kvbm_route_unit* units,
                                                       size_t num_units, int layer_begin, int layer_end, uint32_t src_row_bytes,
                                                       int cast_mode, const float* cast_scales, const kvbm_permute_stream* st,
                                                       cudaStream_t stream)
{
  return repage_gather_batch<kRouted>(srcs, num_srcs, src_page_size, dst, dst_num_heads, dst_page_size, seqs, num_seqs, units, num_units,
                                      layer_begin, layer_end, src_row_bytes, cast_mode, cast_scales, true, st, nullptr, 0, nullptr, 0,
                                      stream);
}

extern "C" cudaError_t
kvbm_kernels_paged_stage_repage_gather_routed_anypage(const kvbm_stage_source* srcs, int num_srcs, uint32_t src_page_size,
                                                      const kvbm_permute_side* dst, uint32_t dst_num_heads, uint32_t dst_page_size,
                                                      const kvbm_route_seq* seqs, size_t num_seqs, const kvbm_route_anypage_unit* units,
                                                      size_t num_units, int layer_begin, int layer_end, uint32_t src_row_bytes, int cast_mode,
                                                      const float* cast_scales, uint32_t* done_flag, uint32_t epoch, uint32_t* completion_flag,
                                                      uint32_t completion_value, cudaStream_t stream)
{
  return repage_gather_batch<kRoutedPhased>(srcs, num_srcs, src_page_size, dst, dst_num_heads, dst_page_size, seqs, num_seqs, units,
                                            num_units, layer_begin, layer_end, src_row_bytes, cast_mode, cast_scales, false, nullptr,
                                            done_flag, epoch, completion_flag, completion_value, stream);
}

extern "C" cudaError_t
kvbm_kernels_paged_stage_repage_gather_routed_anypage_streamed(const kvbm_stage_source* srcs, int num_srcs, uint32_t src_page_size,
                                                               const kvbm_permute_side* dst, uint32_t dst_num_heads, uint32_t dst_page_size,
                                                               const kvbm_route_seq* seqs, size_t num_seqs,
                                                               const kvbm_route_anypage_unit* units, size_t num_units, int layer_begin,
                                                               int layer_end, uint32_t src_row_bytes, int cast_mode, const float* cast_scales,
                                                               const kvbm_permute_stream* st, cudaStream_t stream)
{
  return repage_gather_batch<kRoutedPhased>(srcs, num_srcs, src_page_size, dst, dst_num_heads, dst_page_size, seqs, num_seqs, units,
                                            num_units, layer_begin, layer_end, src_row_bytes, cast_mode, cast_scales, true, st, nullptr, 0,
                                            nullptr, 0, stream);
}

extern "C" cudaError_t
kvbm_kernels_paged_repage_scatter(const kvbm_permute_side* src, uint32_t src_num_heads, uint32_t src_page_size, const kvbm_scatter_target* targets,
                                  int num_targets, uint32_t dst_page_size, uint32_t token_begin, uint32_t token_end, int layer_begin,
                                  int layer_end, uint32_t src_row_bytes, int cast_mode, const float* cast_scales, uint32_t epoch,
                                  uint32_t* completion_flag, uint32_t completion_value, cudaStream_t stream)
{
  return launch_paged_repage_scatter(src, src_num_heads, src_page_size, targets, num_targets, dst_page_size, token_begin, token_end, layer_begin,
                                     layer_end, src_row_bytes, cast_mode, cast_scales, epoch, completion_flag, completion_value, stream);
}

extern "C" cudaError_t
kvbm_kernels_paged_repage_scatter_streamed(const kvbm_permute_side* src, uint32_t src_num_heads, uint32_t src_page_size,
                                           const kvbm_scatter_target* targets, int num_targets, uint32_t dst_page_size, uint32_t token_begin,
                                           uint32_t token_end, int layer_begin, int layer_end, uint32_t src_row_bytes, int cast_mode,
                                           const float* cast_scales, const kvbm_permute_stream* st, cudaStream_t stream)
{
  if (!stream_args_ok(st, 1)) return cudaErrorInvalidValue;
  return launch_paged_repage_scatter(src, src_num_heads, src_page_size, targets, num_targets, dst_page_size, token_begin, token_end, layer_begin,
                                     layer_end, src_row_bytes, cast_mode, cast_scales, st->epoch, st->completion_flag, st->completion_value,
                                     stream, st);
}

extern "C" cudaError_t
kvbm_kernels_paged_repage_scatter_batch(const kvbm_permute_side* src, uint32_t src_num_heads, uint32_t src_page_size,
                                        const kvbm_scatter_target* targets, int num_targets, uint32_t dst_page_size, const kvbm_repage_seq* seqs,
                                        size_t num_seqs, const kvbm_repage_unit* units, size_t num_units, int layer_begin, int layer_end,
                                        uint32_t src_row_bytes, int cast_mode, const float* cast_scales, uint32_t epoch,
                                        uint32_t* completion_flag, uint32_t completion_value, cudaStream_t stream)
{
  return repage_scatter_batch<kSeqs>(src, src_num_heads, src_page_size, targets, num_targets, dst_page_size, seqs, num_seqs, units,
                                     num_units, layer_begin, layer_end, src_row_bytes, cast_mode, cast_scales, false, nullptr, epoch,
                                     completion_flag, completion_value, stream);
}

extern "C" cudaError_t
kvbm_kernels_paged_repage_scatter_batch_streamed(const kvbm_permute_side* src, uint32_t src_num_heads, uint32_t src_page_size,
                                                 const kvbm_scatter_target* targets, int num_targets, uint32_t dst_page_size,
                                                 const kvbm_repage_seq* seqs, size_t num_seqs, const kvbm_repage_unit* units, size_t num_units,
                                                 int layer_begin, int layer_end, uint32_t src_row_bytes, int cast_mode, const float* cast_scales,
                                                 const kvbm_permute_stream* st, cudaStream_t stream)
{
  return repage_scatter_batch<kSeqs>(src, src_num_heads, src_page_size, targets, num_targets, dst_page_size, seqs, num_seqs, units,
                                     num_units, layer_begin, layer_end, src_row_bytes, cast_mode, cast_scales, true, st, 0, nullptr, 0,
                                     stream);
}

extern "C" cudaError_t
kvbm_kernels_paged_repage_scatter_anypage(const kvbm_permute_side* src, uint32_t src_num_heads, uint32_t src_page_size,
                                          const kvbm_scatter_target* targets, int num_targets, uint32_t dst_page_size, const kvbm_repage_seq* seqs,
                                          size_t num_seqs, const kvbm_repage_anypage_unit* units, size_t num_units, int layer_begin,
                                          int layer_end, uint32_t src_row_bytes, int cast_mode, const float* cast_scales, uint32_t epoch,
                                          uint32_t* completion_flag, uint32_t completion_value, cudaStream_t stream)
{
  return repage_scatter_batch<kPhased>(src, src_num_heads, src_page_size, targets, num_targets, dst_page_size, seqs, num_seqs, units,
                                       num_units, layer_begin, layer_end, src_row_bytes, cast_mode, cast_scales, false, nullptr, epoch,
                                       completion_flag, completion_value, stream);
}

extern "C" cudaError_t
kvbm_kernels_paged_repage_scatter_anypage_streamed(const kvbm_permute_side* src, uint32_t src_num_heads, uint32_t src_page_size,
                                                   const kvbm_scatter_target* targets, int num_targets, uint32_t dst_page_size,
                                                   const kvbm_repage_seq* seqs, size_t num_seqs, const kvbm_repage_anypage_unit* units,
                                                   size_t num_units, int layer_begin, int layer_end, uint32_t src_row_bytes, int cast_mode,
                                                   const float* cast_scales, const kvbm_permute_stream* st, cudaStream_t stream)
{
  return repage_scatter_batch<kPhased>(src, src_num_heads, src_page_size, targets, num_targets, dst_page_size, seqs, num_seqs, units,
                                       num_units, layer_begin, layer_end, src_row_bytes, cast_mode, cast_scales, true, st, 0, nullptr, 0,
                                       stream);
}

extern "C" cudaError_t
kvbm_kernels_paged_repage_scatter_routed(const kvbm_permute_side* src, uint32_t src_num_heads, uint32_t src_page_size,
                                         const kvbm_scatter_target* targets, int num_targets, uint32_t dst_page_size, const kvbm_route_seq* seqs,
                                         size_t num_seqs, const kvbm_route_unit* units, size_t num_units, int layer_begin, int layer_end,
                                         uint32_t src_row_bytes, int cast_mode, const float* cast_scales, uint32_t epoch,
                                         uint32_t* completion_flag, uint32_t completion_value, cudaStream_t stream)
{
  return repage_scatter_batch<kRouted>(src, src_num_heads, src_page_size, targets, num_targets, dst_page_size, seqs, num_seqs, units,
                                       num_units, layer_begin, layer_end, src_row_bytes, cast_mode, cast_scales, false, nullptr, epoch,
                                       completion_flag, completion_value, stream);
}

extern "C" cudaError_t
kvbm_kernels_paged_repage_scatter_routed_streamed(const kvbm_permute_side* src, uint32_t src_num_heads, uint32_t src_page_size,
                                                  const kvbm_scatter_target* targets, int num_targets, uint32_t dst_page_size,
                                                  const kvbm_route_seq* seqs, size_t num_seqs, const kvbm_route_unit* units, size_t num_units,
                                                  int layer_begin, int layer_end, uint32_t src_row_bytes, int cast_mode, const float* cast_scales,
                                                  const kvbm_permute_stream* st, cudaStream_t stream)
{
  return repage_scatter_batch<kRouted>(src, src_num_heads, src_page_size, targets, num_targets, dst_page_size, seqs, num_seqs, units,
                                       num_units, layer_begin, layer_end, src_row_bytes, cast_mode, cast_scales, true, st, 0, nullptr, 0,
                                       stream);
}

extern "C" cudaError_t
kvbm_kernels_paged_repage_scatter_routed_anypage(const kvbm_permute_side* src, uint32_t src_num_heads, uint32_t src_page_size,
                                                 const kvbm_scatter_target* targets, int num_targets, uint32_t dst_page_size,
                                                 const kvbm_route_seq* seqs, size_t num_seqs, const kvbm_route_anypage_unit* units,
                                                 size_t num_units, int layer_begin, int layer_end, uint32_t src_row_bytes, int cast_mode,
                                                 const float* cast_scales, uint32_t epoch, uint32_t* completion_flag,
                                                 uint32_t completion_value, cudaStream_t stream)
{
  return repage_scatter_batch<kRoutedPhased>(src, src_num_heads, src_page_size, targets, num_targets, dst_page_size, seqs, num_seqs, units,
                                             num_units, layer_begin, layer_end, src_row_bytes, cast_mode, cast_scales, false, nullptr,
                                             epoch, completion_flag, completion_value, stream);
}

extern "C" cudaError_t
kvbm_kernels_paged_repage_scatter_routed_anypage_streamed(const kvbm_permute_side* src, uint32_t src_num_heads, uint32_t src_page_size,
                                                          const kvbm_scatter_target* targets, int num_targets, uint32_t dst_page_size,
                                                          const kvbm_route_seq* seqs, size_t num_seqs, const kvbm_route_anypage_unit* units,
                                                          size_t num_units, int layer_begin, int layer_end, uint32_t src_row_bytes,
                                                          int cast_mode, const float* cast_scales, const kvbm_permute_stream* st,
                                                          cudaStream_t stream)
{
  return repage_scatter_batch<kRoutedPhased>(src, src_num_heads, src_page_size, targets, num_targets, dst_page_size, seqs, num_seqs, units,
                                             num_units, layer_begin, layer_end, src_row_bytes, cast_mode, cast_scales, true, st, 0, nullptr,
                                             0, stream);
}

extern "C" cudaError_t
kvbm_kernels_paged_stage_gather(const kvbm_stage_source* srcs, int num_srcs, const kvbm_permute_side* dst, uint32_t dst_num_heads,
                                int num_blocks, int layer_begin, int layer_end, uint32_t page_size, uint32_t src_row_bytes, int cast_mode,
                                const float* cast_scales, uint32_t* done_flag, uint32_t epoch, uint32_t* completion_flag,
                                uint32_t completion_value, cudaStream_t stream)
{
  return launch_paged_permute(srcs, num_srcs, dst, dst_num_heads, num_blocks, layer_begin, layer_end, page_size, src_row_bytes, cast_mode,
                              cast_scales, done_flag, epoch, completion_flag, completion_value, KVBM_GATHER_MAX_HEADS, stream);
}

extern "C" cudaError_t
kvbm_kernels_paged_stage_gather_streamed(const kvbm_stage_source* srcs, int num_srcs, const kvbm_permute_side* dst, uint32_t dst_num_heads,
                                         int num_blocks, int layer_begin, int layer_end, uint32_t page_size, uint32_t src_row_bytes,
                                         int cast_mode, const float* cast_scales, const kvbm_permute_stream* st, cudaStream_t stream)
{
  if (!stream_args_ok(st, num_srcs)) return cudaErrorInvalidValue;
  return launch_paged_permute(srcs, num_srcs, dst, dst_num_heads, num_blocks, layer_begin, layer_end, page_size, src_row_bytes, cast_mode,
                              cast_scales, st->done_flag, st->epoch, st->completion_flag, st->completion_value, KVBM_GATHER_MAX_HEADS, stream,
                              st);
}

extern "C" cudaError_t
kvbm_kernels_paged_repage_gather_streamed(const kvbm_permute_source* srcs, int num_srcs, uint32_t src_page_size, const kvbm_permute_side* dst,
                                          uint32_t dst_num_heads, uint32_t dst_page_size, uint32_t token_begin, uint32_t token_end,
                                          int layer_begin, int layer_end, uint32_t src_row_bytes, int cast_mode, const float* cast_scales,
                                          const kvbm_permute_stream* st, cudaStream_t stream)
{
  if (!stream_args_ok(st, num_srcs)) return cudaErrorInvalidValue;
  kvbm_stage_source staged[KVBM_GATHER_MAX_SOURCES];
  return launch_paged_repage_gather(one_stage(srcs, num_srcs, dst, staged), num_srcs, src_page_size, dst, dst_num_heads, dst_page_size,
                                    token_begin, token_end, layer_begin, layer_end, src_row_bytes, cast_mode, cast_scales, st->done_flag,
                                    st->epoch, st->completion_flag, st->completion_value, KVBM_GATHER_MAX_HEADS, stream, st);
}

extern "C" bool
kvbm_kernels_has_memcpy_batch_async(void)
{
#if CUDART_VERSION >= 12090
  return true;
#else
  return false;
#endif
}

extern "C" bool
kvbm_kernels_is_stub_build(void)
{
  return false;
}

// =================================================================================================
// C ABI -- Part 2 (v2 extensions)
// =================================================================================================
static cudaError_t
paged_copy_impl(const kvbm_paged_layout* src, const kvbm_paged_dst* dsts, int num_dsts, int num_blocks,
                int layer_begin, int layer_end, int cast_mode, const kvbm_paged_copy_opts* opts,
                cudaStream_t stream)
{
  if (num_blocks == 0 || num_dsts == 0 || layer_end == layer_begin) return cudaSuccess;
  if (!src || !dsts) return cudaErrorInvalidValue;
  if (num_blocks < 0 || num_dsts < 0 || num_dsts > KVBM_MAX_DESTINATIONS) return cudaErrorInvalidValue;
  if (layer_begin < 0 || layer_end < layer_begin || static_cast<uint32_t>(layer_end) > src->num_layers)
    return cudaErrorInvalidValue;
  if (cast_mode < KVBM_CAST_NONE || cast_mode > KVBM_CAST_BF16_TO_FP8E4M3) return cudaErrorInvalidValue;
  if (!src->layer_base || src->region_bytes == 0) return cudaErrorInvalidValue;
  const uint32_t num = cast_mode == KVBM_CAST_FP8E4M3_TO_BF16 ? 2 : 1;
  const uint32_t den = cast_mode == KVBM_CAST_BF16_TO_FP8E4M3 ? 2 : 1;
  if (cast_mode == KVBM_CAST_BF16_TO_FP8E4M3 && (src->region_bytes & 1)) return cudaErrorInvalidValue;

  kvbm_paged_copy_opts o{};
  if (opts) o = *opts;

  // NVLS: dsts[0] is addressed through a multicast mapping and carries the payload for every bound device; the
  // other entries only name the flags of the remaining receivers.
  const bool mc = o.multicast != 0;
  if (mc && (cast_mode != KVBM_CAST_NONE || (src->region_bytes & 3) || (src->block_stride & 3) || (src->outer_stride & 3) ||
             (dsts[0].layout.block_stride & 15) || (dsts[0].layout.outer_stride & 15)))
    return cudaErrorInvalidValue;
  const int data_dsts = mc ? 1 : num_dsts;

  // a scaled cast packs the outer index above the layer of every item (CastScales)
  const float* scales = o.cast_scales;
  if (scales && (src->num_layers > 65536 || src->outer_dim > 32768)) return cudaErrorInvalidValue;

  PagedGen<false> gen{};
  PagedSyncArgs sync{};
  gen.a.src = *src;
  gen.a.ndst = data_dsts;
  gen.a.replicate = 1;
  sync.num_flag_dsts = num_dsts;
  for (int d = 0; d < num_dsts; ++d) {
    const kvbm_paged_dst& D = dsts[d];
    sync.done_flag[d] = D.done_flag;
    sync.layer_done[d] = D.layer_done_flags;
    if (d >= data_dsts) continue;
    // same compatibility rules as execute_cuda_transfer (executor/cuda.rs:52-67) + region size match
    // (executor/memcpy.rs:143-153), adjusted for the element-width change of a cast
    if (!D.layout.layer_base || !D.src_block_ids || !D.dst_block_ids) return cudaErrorInvalidValue;
    if (D.layout.num_layers != src->num_layers || D.layout.outer_dim != src->outer_dim) return cudaErrorInvalidValue;
    if (static_cast<uint64_t>(D.layout.region_bytes) * den != static_cast<uint64_t>(src->region_bytes) * num)
      return cudaErrorInvalidValue;
    gen.a.dst[d] = D.layout;
    gen.a.src_ids[d] = D.src_block_ids;
    gen.a.dst_ids[d] = D.dst_block_ids;
    if (D.src_block_ids != dsts[0].src_block_ids) gen.a.replicate = 0;
  }
  if (data_dsts == 1) gen.a.replicate = 1;
  sync.completion_flag = o.completion_flag;
  sync.completion_value = o.completion_value;
  sync.layer_ready = o.layer_ready_flags;
  sync.epoch = o.epoch;
  sync.gate_timeout_ns = static_cast<uint64_t>(o.gate_timeout_ms > 0 ? o.gate_timeout_ms : 10000) * 1000000ull;
  if (o.layer_ready_flags && !o.sync_workspace) return cudaErrorInvalidValue;  // the abort word lives in the workspace
  bool needs_ws = o.completion_flag != nullptr;
  for (int d = 0; d < num_dsts; ++d)
    if (dsts[d].done_flag || dsts[d].layer_done_flags) needs_ws = true;
  if (needs_ws && !o.sync_workspace) return cudaErrorInvalidValue;

  DeviceInfo di;
  cudaError_t e = device_info(&di);
  if (e != cudaSuccess) return e;
  RingCfg rc = make_ring(di, src->region_bytes, o.warps_per_cta, o.stages, o.tile_bytes, cast_mode, o.stores_in_flight);

  gen.a.n_blocks = static_cast<uint32_t>(num_blocks);
  gen.a.layer_begin = static_cast<uint32_t>(layer_begin);
  gen.a.n_layers = static_cast<uint32_t>(layer_end - layer_begin);
  gen.a.outer = src->outer_dim;
  gen.a.tile = rc.tile;
  // in 64 bits: a region within one tile of 4 GiB would wrap to 0 tiles in 32
  gen.a.tiles_per_region = static_cast<uint32_t>((static_cast<uint64_t>(src->region_bytes) + rc.tile - 1) / rc.tile);
  gen.a.dst_num = num;
  gen.a.dst_den = den;
  const uint64_t fan = gen.a.replicate ? 1 : static_cast<uint64_t>(data_dsts);
  const uint64_t total = static_cast<uint64_t>(gen.a.n_layers) * gen.a.n_blocks * gen.a.outer * fan * gen.a.tiles_per_region;
  if (total >= (1ull << 31)) return cudaErrorInvalidValue;

  const uint64_t rings_needed = (total + rc.batch - 1) / rc.batch;
  const uint64_t ctas_needed = (rings_needed + rc.rings - 1) / rc.rings;
  // Default: one CTA per SM (see the note at kDefaultTile); max_ctas leaves SMs to whatever the engine is running.
  int cap = o.max_ctas > 0 ? o.max_ctas : default_ctas(di);
  const int grid = static_cast<int>(std::min<uint64_t>(ctas_needed, static_cast<uint64_t>(cap)));
  const int allow_tma = o.force_simt ? 0 : 1;
  const uint32_t total32 = static_cast<uint32_t>(total);

  // control words: the caller's workspace ([num_layers] layer counters, then 3 control words) or a pool slot
  int dev = 0, pool_slot = -1;
  if (o.sync_workspace) {
    sync.layer_counters = o.sync_workspace;
    sync.ctl = o.sync_workspace + src->num_layers;
  } else if (!o.static_schedule && cudaGetDevice(&dev) == cudaSuccess && dev >= 0 && dev < 64) {
    sync.ctl = sched_acquire(dev, stream, &pool_slot);
  }

  auto launch = [&](auto kern, const auto& g) -> cudaError_t {
    cudaError_t err = set_smem(kern, rc.smem);
    if (err == cudaSuccess) {
      kern<<<grid, rc.rings * 64, rc.smem, stream>>>(g, sync, total32, rc.stages, rc.pending, rc.batch, o.static_schedule,
                                                     rc.out_tile, allow_tma, o.cache_hint, mc ? (o.multicast == 2 ? 0 : 4) : o.variant, scales);
      g_launches.fetch_add(1, std::memory_order_relaxed);
      err = cudaGetLastError();
    }
    sched_release(dev, pool_slot, stream);
    return err;
  };
  // the plain hot path gets the kernel with the generality folded away at compile time (copy_engine.cuh, FAST)
  bool any_layer_flags = false;
  for (int d = 0; d < num_dsts; ++d) any_layer_flags = any_layer_flags || dsts[d].layer_done_flags != nullptr;
  const bool fast = !mc && o.variant == 0 && o.cache_hint == 0 && allow_tma && !o.layer_ready_flags && !any_layer_flags &&
                    (gen.a.replicate ? data_dsts : 1) == 1;
  // a scaled cast takes the general rings (its own instantiation), whatever `fast` says
  const PagedGen<true> sgen{gen.a};
  switch (cast_mode) {
    case KVBM_CAST_NONE:
      return fast ? launch(kvbm_paged_copy_kernel<KVBM_CAST_NONE, true>, gen) : launch(kvbm_paged_copy_kernel<KVBM_CAST_NONE, false>, gen);
    case KVBM_CAST_FP8E4M3_TO_BF16:
      if (scales) return launch(kvbm_paged_copy_kernel<KVBM_CAST_FP8E4M3_TO_BF16, false, true>, sgen);
      return fast ? launch(kvbm_paged_copy_kernel<KVBM_CAST_FP8E4M3_TO_BF16, true>, gen) : launch(kvbm_paged_copy_kernel<KVBM_CAST_FP8E4M3_TO_BF16, false>, gen);
    default:
      if (scales) return launch(kvbm_paged_copy_kernel<KVBM_CAST_BF16_TO_FP8E4M3, false, true>, sgen);
      return fast ? launch(kvbm_paged_copy_kernel<KVBM_CAST_BF16_TO_FP8E4M3, true>, gen) : launch(kvbm_paged_copy_kernel<KVBM_CAST_BF16_TO_FP8E4M3, false>, gen);
  }
}

// CUDA loads modules lazily by default, and the first launch of a not-yet-loaded kernel (of ANY module in the process)
// can wait for the device to drain -- which never happens while a gated transfer spins on ready flags that the stalled
// launch was supposed to release.  This library preloads its own kernels, but it cannot load the engine's.  So a
// spinning gate is only used when the process runs with eager loading (or the caller insists); otherwise the gate
// moves to the stream front-end: one cuStreamWaitValue32 + one single-layer launch per layer -- nothing resident spins.
static bool eager_module_loading()
{
  static const int mode = [] {
    typedef int (*fn_t)(int*);
    void* f = nullptr;
    cudaDriverEntryPointQueryResult r;
    int m = 0;
    if (cudaGetDriverEntryPoint("cuModuleGetLoadingMode", &f, cudaEnableDefault, &r) == cudaSuccess && f &&
        reinterpret_cast<fn_t>(f)(&m) == 0)
      return m;
    (void)cudaGetLastError();
    return 0;
  }();
  return mode == 1;  // CU_MODULE_EAGER_LOADING
}

extern "C" int
kvbm_kernels_gate_would_spin(void)
{
  return eager_module_loading() ? 1 : 0;
}

extern "C" cudaError_t
kvbm_kernels_paged_copy_v2(const kvbm_paged_layout* src, const kvbm_paged_dst* dsts, int num_dsts, int num_blocks,
                           int layer_begin, int layer_end, int cast_mode, const kvbm_paged_copy_opts* opts,
                           cudaStream_t stream)
{
  if (opts && opts->cast_scales && cast_mode == KVBM_CAST_NONE) return cudaErrorInvalidValue;  // scales belong to a cast's fp8 side
  const bool gated = opts && opts->layer_ready_flags != nullptr;
  if (!gated || num_blocks == 0 || num_dsts == 0 || layer_end <= layer_begin || !dsts || num_dsts < 0 || num_dsts > KVBM_MAX_DESTINATIONS)
    return paged_copy_impl(src, dsts, num_dsts, num_blocks, layer_begin, layer_end, cast_mode, opts, stream);
  const int mode = opts->gate_mode;
  if (mode < KVBM_GATE_AUTO || mode > KVBM_GATE_STREAM_WAIT) return cudaErrorInvalidValue;
  if (mode == KVBM_GATE_SPIN || (mode == KVBM_GATE_AUTO && eager_module_loading()))
    return paged_copy_impl(src, dsts, num_dsts, num_blocks, layer_begin, layer_end, cast_mode, opts, stream);
  DeviceInfo di;
  cudaError_t e = device_info(&di);
  if (e != cudaSuccess) return e;
  if (!stream_memops()) return mode == KVBM_GATE_AUTO ? paged_copy_impl(src, dsts, num_dsts, num_blocks, layer_begin, layer_end, cast_mode, opts, stream)
                                                       : cudaErrorNotSupported;
  kvbm_paged_copy_opts o = *opts;
  o.layer_ready_flags = nullptr;
  kvbm_paged_dst dd[KVBM_MAX_DESTINATIONS];
  for (int l = layer_begin; l < layer_end; ++l) {
    const bool last = l + 1 == layer_end;
    // CU_STREAM_WAIT_VALUE_GEQ: the stream front-end polls the word, no SM is occupied; (int32)(flag - epoch) >= 0, the order
    // the spinning gate uses too (epoch_reached)
    if (g_wait32(stream, reinterpret_cast<unsigned long long>(opts->layer_ready_flags + l), opts->epoch, 0) != 0) return cudaErrorUnknown;
    for (int d = 0; d < num_dsts; ++d) {
      dd[d] = dsts[d];
      if (!last) dd[d].done_flag = nullptr;
    }
    o.completion_flag = last ? opts->completion_flag : nullptr;
    if ((e = paged_copy_impl(src, dd, num_dsts, num_blocks, l, l + 1, cast_mode, &o, stream)) != cudaSuccess) return e;
  }
  return cudaSuccess;
}

extern "C" cudaError_t
kvbm_kernels_set_flags(uint32_t* flags, int first, int count, uint32_t value, cudaStream_t stream)
{
  if (count == 0) return cudaSuccess;
  if (!flags || count < 0 || first < 0) return cudaErrorInvalidValue;
  DeviceInfo di;
  cudaError_t e = device_info(&di);
  if (e != cudaSuccess) return e;
  if (count == 1 && stream_memops()) {
    // CU_STREAM_WRITE_VALUE_DEFAULT (0): memory fence before the write => release semantics for prior work
    if (g_write32(stream, reinterpret_cast<unsigned long long>(flags + first), value, 0) == 0) return cudaSuccess;
  }
  kvbm_set_flags_kernel<<<(count + 127) / 128, 128, 0, stream>>>(flags, first, count, value);
  g_launches.fetch_add(1, std::memory_order_relaxed);
  return cudaGetLastError();
}

extern "C" cudaError_t
kvbm_kernels_wait_flag(const uint32_t* flag, uint32_t value, cudaStream_t stream)
{
  if (!flag) return cudaErrorInvalidValue;
  DeviceInfo di;
  cudaError_t e = device_info(&di);
  if (e != cudaSuccess) return e;
  if (stream_memops()) {
    // CU_STREAM_WAIT_VALUE_GEQ (0): wait until (int32)(*flag - value) >= 0
    if (g_wait32(stream, reinterpret_cast<unsigned long long>(flag), value, 0) == 0) return cudaSuccess;
  }
  kvbm_wait_flag_kernel<<<1, 1, 0, stream>>>(flag, value);
  g_launches.fetch_add(1, std::memory_order_relaxed);
  return cudaGetLastError();
}

extern "C" cudaError_t
kvbm_kernels_stream_wait_event(cudaStream_t stream, void* event)
{
  if (!event) return cudaErrorInvalidValue;
  return cudaStreamWaitEvent(stream, static_cast<cudaEvent_t>(event), 0);
}

extern "C" uint64_t
kvbm_kernels_launch_count(void)
{
  return g_launches.load(std::memory_order_relaxed);
}

extern "C" const char*
kvbm_kernels_build_info(void)
{
  return "libkvbm_kernels sm_90a tma=cp.async.bulk cast=e4m3<->bf16";
}
