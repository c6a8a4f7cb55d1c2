// libkvbm_physical.so -- host half of the KV transfer path (C++ restatement of Dynamo's kvbm-physical crate
// for this path; see include/kvbm_physical.h for the reference lines every entry point replaces).
#include <cuda_runtime_api.h>

#include <atomic>
#include <chrono>
#include <cstdlib>
#include <cstring>
#include <algorithm>
#include <memory>
#include <mutex>
#include <random>
#include <set>
#include <string>
#include <thread>
#include <unordered_map>
#include <unordered_set>
#include <vector>

#include <sched.h>
#include <unistd.h>

#include "layout.hpp"
#include "serialized_layout.hpp"

namespace kvbm_host {

static thread_local std::string g_last_error;

// Identity of this address space for layout blobs: the pid alone collides across PID namespaces (two containers can
// both be pid 1), so a per-process random nonce rides in the upper 32 bits of the header's pid field.
static uint64_t process_identity()
{
  static const uint64_t id = [] {
    std::random_device rd;
    uint64_t nonce = (static_cast<uint64_t>(rd()) << 32 | rd()) ^
                     static_cast<uint64_t>(std::chrono::steady_clock::now().time_since_epoch().count());
    nonce ^= nonce >> 29;
    return (static_cast<uint64_t>(getpid()) & 0xffffffffull) | ((nonce & 0xffffffffull) << 32);
  }();
  return id;
}

static int fail(int code, const std::string& msg)
{
  g_last_error = msg;
  return code;
}
int set_last_error(int code, const std::string& msg) { return fail(code, msg); }
static int fail_cuda(cudaError_t e, const char* what)
{
  g_last_error = std::string(what) + " failed: " + cudaGetErrorName(e) + " (" + std::to_string(static_cast<int>(e)) + ")";
  (void)cudaGetLastError();
  return KVBM_ERR_CUDA;
}
#define CU(call)                                   \
  do {                                             \
    cudaError_t e__ = (call);                      \
    if (e__ != cudaSuccess) return fail_cuda(e__, #call); \
  } while (0)

// ---------------------------------------------------------------------------------------------------
// validation.rs
// ---------------------------------------------------------------------------------------------------
// Fast path of the three checks below for the common case (every id in range): one bitmap over the destination's
// block ids instead of a hash set -- 256 ids cost ~0.3 us instead of ~10 us, which is a tenth of a whole 512 MiB
// same-GPU transfer.  Returns false when anything is wrong (or an id is out of range); the reference-ordered slow
// path then produces the exact error.
static bool validate_fast(const size_t* src_ids, const size_t* dst_ids, size_t n, size_t src_blocks, size_t dst_blocks,
                          bool same_layout)
{
  thread_local std::vector<uint64_t> bits;
  const size_t words = (dst_blocks + 63) / 64;
  if (words > (1u << 20)) return false;  // absurdly large pools: take the general path
  if (bits.size() < words) bits.resize(words, 0);
  bool ok = true;
  size_t marked = 0;
  for (; marked < n; ++marked) {
    const size_t d = dst_ids[marked];
    if (d >= dst_blocks || src_ids[marked] >= src_blocks) {
      ok = false;
      break;
    }
    uint64_t& w = bits[d >> 6];
    const uint64_t m = 1ull << (d & 63);
    if (w & m) {
      ok = false;
      break;
    }
    w |= m;
  }
  if (ok && same_layout)
    for (size_t i = 0; i < n; ++i) {
      const size_t v = src_ids[i];
      if (v < dst_blocks && (bits[v >> 6] >> (v & 63)) & 1) {
        ok = false;
        break;
      }
    }
  for (size_t i = 0; i < marked; ++i) bits[dst_ids[i] >> 6] = 0;  // leave the scratch bitmap clean
  return ok;
}

// The id checks of validate_block_transfer in its order, for lists of any lengths (a re-paging transfer's two lists differ).
static int check_block_ids(const size_t* src_ids, size_t n_src, const size_t* dst_ids, size_t n_dst, size_t src_blocks,
                           size_t dst_blocks, bool same_layout)
{
  std::unordered_set<size_t> seen;
  seen.reserve(n_dst * 2);
  for (size_t i = 0; i < n_dst; ++i)  // validate_dst_unique, validation.rs:55-70
    if (!seen.insert(dst_ids[i]).second)
      return fail(KVBM_ERR_DUPLICATE_DST, "Destination block IDs are not unique: duplicates = [" + std::to_string(dst_ids[i]) + "]");
  if (same_layout) {  // validate_disjoint_same_layout, validation.rs:112-136
    for (size_t i = 0; i < n_src; ++i)
      if (seen.count(src_ids[i]))
        return fail(KVBM_ERR_OVERLAP, "Source and destination blocks overlap (same layout): overlapping = [" + std::to_string(src_ids[i]) + "]");
  }
  for (size_t i = 0; i < std::max(n_src, n_dst); ++i) {  // validate_block_ids_in_range, validation.rs:139-158
    if (i < n_src && src_ids[i] >= src_blocks)
      return fail(KVBM_ERR_RANGE, "Block ID " + std::to_string(src_ids[i]) + " out of range for source (max=" + std::to_string(src_blocks) + ")");
    if (i < n_dst && dst_ids[i] >= dst_blocks)
      return fail(KVBM_ERR_RANGE, "Block ID " + std::to_string(dst_ids[i]) + " out of range for destination (max=" + std::to_string(dst_blocks) + ")");
  }
  return KVBM_OK;
}

static int validate_block_transfer(const size_t* src_ids, size_t n_src, const size_t* dst_ids, size_t n_dst,
                                   size_t src_blocks, size_t dst_blocks, bool same_layout)
{
  if (n_src != n_dst)  // validation.rs:177-183
    return fail(KVBM_ERR_LENGTH_MISMATCH, "Block ID lists have mismatched lengths: src=" + std::to_string(n_src) +
                                              ", dst=" + std::to_string(n_dst) + ", bounce=None");
  if (n_src == 0 || validate_fast(src_ids, dst_ids, n_src, src_blocks, dst_blocks, same_layout)) return KVBM_OK;
  return check_block_ids(src_ids, n_src, dst_ids, n_dst, src_blocks, dst_blocks, same_layout);
}

// ---------------------------------------------------------------------------------------------------
// strategy.rs:138-210 (local-to-local rows).  Device index is ignored exactly like strategy.rs:168.
// ---------------------------------------------------------------------------------------------------
// select_remote_strategy (strategy.rs:213-243): the source is local, the destination another agent's
static int select_remote_strategy(int src, const kvbm_transfer_capabilities* caps, kvbm_transfer_plan* out)
{
  if (src == KVBM_STORAGE_SYSTEM || src == KVBM_STORAGE_PINNED) {
    *out = kvbm_transfer_plan{0, KVBM_STRATEGY_NIXL_WRITE, 0, KVBM_STRATEGY_INVALID};
  } else if (src == KVBM_STORAGE_DEVICE) {
    if (caps && caps->allow_gpu_rdma)
      *out = kvbm_transfer_plan{0, KVBM_STRATEGY_NIXL_WRITE, 0, KVBM_STRATEGY_INVALID};
    else
      *out = kvbm_transfer_plan{1, KVBM_STRATEGY_CUDA_ASYNC_D2H, KVBM_STORAGE_PINNED, KVBM_STRATEGY_NIXL_WRITE};
  } else {
    *out = kvbm_transfer_plan{1, KVBM_STRATEGY_NIXL_WRITE, KVBM_STORAGE_PINNED, KVBM_STRATEGY_NIXL_WRITE};  // Disk -> Remote
  }
  return KVBM_OK;
}

static int select_direct_strategy(int src, int dst, const kvbm_transfer_capabilities* caps, kvbm_transfer_plan* out, bool dst_is_remote = false)
{
  if (dst_is_remote) {  // strategy.rs:147-150
    if (src < 0 || src > KVBM_STORAGE_DISK || dst < 0 || dst > KVBM_STORAGE_DISK) return fail(KVBM_ERR, "unknown StorageKind");
    return select_remote_strategy(src, caps, out);
  }
  auto direct = [&](int s) {
    *out = kvbm_transfer_plan{0, s, 0, KVBM_STRATEGY_INVALID};
    return KVBM_OK;
  };
  auto two_hop = [&](int first, int second) {
    *out = kvbm_transfer_plan{1, first, KVBM_STORAGE_PINNED, second};
    return KVBM_OK;
  };
  const bool gds = caps && caps->allow_gds;
  const bool host_s = src == KVBM_STORAGE_SYSTEM || src == KVBM_STORAGE_PINNED;
  const bool host_d = dst == KVBM_STORAGE_SYSTEM || dst == KVBM_STORAGE_PINNED;
  if (src < 0 || src > KVBM_STORAGE_DISK || dst < 0 || dst > KVBM_STORAGE_DISK) return fail(KVBM_ERR, "unknown StorageKind");
  if (host_s && host_d) return direct(KVBM_STRATEGY_MEMCPY);
  if (src == KVBM_STORAGE_SYSTEM && dst == KVBM_STORAGE_DEVICE) return fail(KVBM_ERR_UNSUPPORTED, "System to Device transfers are not supported");
  if (src == KVBM_STORAGE_PINNED && dst == KVBM_STORAGE_DEVICE) return direct(KVBM_STRATEGY_CUDA_ASYNC_H2D);
  if (src == KVBM_STORAGE_DEVICE && dst == KVBM_STORAGE_SYSTEM) return fail(KVBM_ERR_UNSUPPORTED, "Device to System transfers are not supported");
  if (src == KVBM_STORAGE_DEVICE && dst == KVBM_STORAGE_PINNED) return direct(KVBM_STRATEGY_CUDA_ASYNC_D2H);
  if (src == KVBM_STORAGE_DEVICE && dst == KVBM_STORAGE_DEVICE) return direct(KVBM_STRATEGY_CUDA_ASYNC_D2D);
  if (host_s && dst == KVBM_STORAGE_DISK) return direct(KVBM_STRATEGY_NIXL_WRITE);
  if (src == KVBM_STORAGE_DISK && host_d) return direct(KVBM_STRATEGY_NIXL_READ_FLIPPED);
  if (src == KVBM_STORAGE_DISK && dst == KVBM_STORAGE_DISK) return two_hop(KVBM_STRATEGY_NIXL_READ_FLIPPED, KVBM_STRATEGY_NIXL_WRITE);
  if (src == KVBM_STORAGE_DEVICE && dst == KVBM_STORAGE_DISK)
    return gds ? direct(KVBM_STRATEGY_NIXL_WRITE) : two_hop(KVBM_STRATEGY_CUDA_ASYNC_D2H, KVBM_STRATEGY_NIXL_WRITE);
  if (src == KVBM_STORAGE_DISK && dst == KVBM_STORAGE_DEVICE)
    return gds ? direct(KVBM_STRATEGY_NIXL_READ) : two_hop(KVBM_STRATEGY_NIXL_READ_FLIPPED, KVBM_STRATEGY_CUDA_ASYNC_H2D);
  return fail(KVBM_ERR, "unreachable strategy");
}

// select_strategy (strategy.rs:78-108) + select_remote_strategy_v2 (:245-281): locality = whose agent owns the layout
static int select_strategy(int src, bool src_local, int dst, bool dst_local, const kvbm_transfer_capabilities* caps, kvbm_transfer_plan* out)
{
  if (src < 0 || src > KVBM_STORAGE_DISK || dst < 0 || dst > KVBM_STORAGE_DISK) return fail(KVBM_ERR, "unknown StorageKind");
  if (!src_local && !dst_local) return fail(KVBM_ERR_UNSUPPORTED, "Both src and dst are remote - this is not supported.");
  if (src_local && dst_local) return select_direct_strategy(src, dst, caps, out);
  if (src == KVBM_STORAGE_DISK || dst == KVBM_STORAGE_DISK)
    return fail(KVBM_ERR_UNSUPPORTED, "Neither local nor remote disk transfers are supported over NIXL at this time.");
  if (!(caps && caps->allow_gpu_rdma) && (src == KVBM_STORAGE_DEVICE || dst == KVBM_STORAGE_DEVICE))
    return fail(KVBM_ERR_UNSUPPORTED, "GPU RDMA is disabled - this transfer requires GPU RDMA.");
  *out = kvbm_transfer_plan{0, src_local ? KVBM_STRATEGY_NIXL_WRITE : KVBM_STRATEGY_NIXL_READ_FLIPPED, 0, KVBM_STRATEGY_INVALID};
  return KVBM_OK;
}

// ---------------------------------------------------------------------------------------------------
// KvBlockLayout::requires_transform (kv_block_layout.rs:107-119) and select_transform_kernel (executor/mod.rs:46-100)
// ---------------------------------------------------------------------------------------------------
static bool kv_known(int k) { return k >= KVBM_KV_UNIVERSAL_TP && k <= KVBM_KV_CUSTOM; }
static bool kv_requires_transform(int a, int b)
{
  if (a == KVBM_KV_CUSTOM || b == KVBM_KV_CUSTOM) return true;  // the int does not carry Custom's dimension order: never assume equality
  if (kv_known(a) && kv_known(b)) return a != b;  // dim orders of the four named formats are pairwise different
  if (!kv_known(a) && !kv_known(b)) return false; // Unknown -> Unknown: compatible (the reference warns)
  return true;                                    // Unknown <-> known: conservative
}
static int select_transform_kernel(int src, int dst)
{
  if (!kv_requires_transform(src, dst)) return KVBM_TRANSFORM_NONE;
  if (!kv_known(src) || !kv_known(dst)) return KVBM_TRANSFORM_UNSUPPORTED;
  const bool s_op = src == KVBM_KV_OPERATIONAL_NHD || src == KVBM_KV_OPERATIONAL_HND;
  const bool d_op = dst == KVBM_KV_OPERATIONAL_NHD || dst == KVBM_KV_OPERATIONAL_HND;
  const bool s_un = src == KVBM_KV_UNIVERSAL_TP || src == KVBM_KV_UNIVERSAL_PP;
  const bool d_un = dst == KVBM_KV_UNIVERSAL_TP || dst == KVBM_KV_UNIVERSAL_PP;
  if (s_op && d_un) return KVBM_TRANSFORM_BLOCK_TO_UNIVERSAL;
  if (s_un && d_op) return KVBM_TRANSFORM_UNIVERSAL_TO_BLOCK;
  if (s_op && d_op) return KVBM_TRANSFORM_OPERATIONAL_TRANSPOSE;
  return KVBM_TRANSFORM_UNSUPPORTED;  // Custom, and Universal <-> Universal (a TODO in the reference, :87-91)
}
static const char* kv_name(int k)
{
  static const char* n[] = {"Unknown", "UniversalTP", "UniversalPP", "OperationalHND", "OperationalNHD", "Custom"};
  return n[k >= 0 && k <= 5 ? k : 0];
}

// ---------------------------------------------------------------------------------------------------
// TransferManager
// ---------------------------------------------------------------------------------------------------
constexpr int kSlots = 64;     // in-flight transfers before the host has to wait for the oldest
constexpr int kStreams = 4;    // context.rs:286-292: 4 h2d + 4 d2h streams, round-robin

struct Slot {
  int32_t* pinned_ids = nullptr;  // staging for the narrowed block tables (H2D source)
  int32_t* dev_ids = nullptr;
  size_t cap = 0;                 // capacity in int32 entries
  uint32_t* host_flag = nullptr;  // mapped pinned word the kernel's last warp writes
  uint32_t* dev_ws = nullptr;     // sync workspace (zeroed, kernel leaves it zeroed)
  size_t ws_cap = 0;
  cudaEvent_t ev = nullptr;
  std::atomic<uint64_t> seq{0};   // owner (read lock-free by kvbm_notification_is_complete)
  bool in_flight = false;
  bool owns_ids = false;          // false: pinned_ids / dev_ids point into the manager's arenas
  bool owns_ws = false;
  bool owns_flag = false;
};
constexpr size_t kArenaIds = 4096;  // int32 entries per slot carved from the arenas (16 KiB: 2 x 2048-block tables)
constexpr size_t kArenaWs = 512;    // workspace words per slot

#pragma pack(push, 1)
struct BlobHeader {
  char magic[8];
  uint32_t version;
  uint32_t fully_contiguous;
  uint32_t block_dim;
  uint32_t storage;
  int32_t device_id;
  uint32_t n_allocs;
  uint64_t worker_id;
  uint64_t pid;
  uint64_t cfg[9];
};
struct BlobAlloc {
  uint64_t addr;
  uint64_t size;
  uint64_t offset_in_ipc;   // addr - base of the cudaMalloc allocation the IPC handle names
  uint32_t has_ipc;
  unsigned char ipc[64];
};
#pragma pack(pop)
constexpr uint32_t kBlobVersion = 1;
static const char kMagic[8] = {'K', 'V', 'B', 'M', 'L', 'A', 'Y', '1'};

}  // namespace kvbm_host

using namespace kvbm_host;

struct kvbm_transfer_manager {
  int device = -1;       // < 0: host-only
  uint64_t worker_id = 0;
  std::mutex mu;
  std::unordered_map<uint64_t, std::unique_ptr<Layout>> layouts;
  uint16_t next_layout_id = 1;
  cudaStream_t h2d[kStreams] = {};
  cudaStream_t d2h[kStreams] = {};
  std::atomic<uint32_t> rr_h2d{0}, rr_d2h{0};
  Slot slots[kSlots];
  // one pinned and one device allocation back all slots (128 cudaHostAlloc + 128 cudaMalloc per manager took seconds
  // on a multi-GPU box); a slot only allocates privately when a transfer outgrows its share
  uint8_t* pinned_arena = nullptr;
  uint8_t* dev_arena = nullptr;
  uint64_t next_seq = 1;
  std::atomic<uint64_t> bytes_moved{0}, h2d_bytes{0};
  // CUDA IPC mappings opened by import_metadata, keyed by the 64-byte handle: an allocation shared by several
  // imported layouts (e.g. two tensors in one allocator segment) is mapped once; closed when the manager dies.
  std::unordered_map<std::string, void*> ipc_cache;
  // other devices whose memory this manager's device may touch: peer access enabled through kvbm_manager_enable_peer_access,
  // or the devices of IPC mappings opened with lazy peer access
  std::set<int> peers;
  // (agent name, worker id) of every SerializedLayout imported so far (manager/mod.rs:572-584 refuses a second load)
  std::set<std::pair<std::string, uint64_t>> loaded_remotes;
  // TransferCapabilities (transfer/strategy.rs:245-278).  allow_gpu_rdma = peers may be written directly over NVLink
  // (the default here); 0 forces the reference's TwoHop plan Device -> Pinned -> Device through a bounce buffer.
  kvbm_transfer_capabilities caps{0, 1};

  Layout* find(kvbm_layout_handle h)
  {
    auto it = layouts.find(h);
    return it == layouts.end() ? nullptr : it->second.get();
  }
};

namespace kvbm_host {

struct DeviceGuard {
  int prev = -1;
  bool active = false;
  explicit DeviceGuard(int dev)
  {
    if (dev >= 0 && cudaGetDevice(&prev) == cudaSuccess && prev != dev) {
      active = cudaSetDevice(dev) == cudaSuccess;
    }
  }
  ~DeviceGuard()
  {
    if (active) cudaSetDevice(prev);
  }
};

static int upload_layer_base(kvbm_transfer_manager* m, Layout* L)
{
  if (m->device < 0) return KVBM_OK;
  DeviceGuard g(m->device);
  CU(cudaMalloc(reinterpret_cast<void**>(&L->dev_layer_base), L->layer_base.size() * sizeof(uint64_t)));
  CU(cudaMemcpy(L->dev_layer_base, L->layer_base.data(), L->layer_base.size() * sizeof(uint64_t), cudaMemcpyHostToDevice));
  return KVBM_OK;
}

// LayoutHandle = (worker_id, layout_id: u16) (manager/handle.rs:16-50).  Ids of unregistered layouts are reused; a live
// layout is never overwritten: 0 = "the 16-bit id space of this worker is exhausted".
static kvbm_layout_handle add_layout(kvbm_transfer_manager* m, Layout&& L)
{
  std::lock_guard<std::mutex> lk(m->mu);
  for (uint32_t tries = 0; tries < 65535; ++tries) {
    uint16_t id = m->next_layout_id++;
    if (id == 0) id = m->next_layout_id++;
    const kvbm_layout_handle h = (m->worker_id << 16) | id;
    if (m->layouts.find(h) != m->layouts.end()) continue;
    m->layouts[h] = std::make_unique<Layout>(std::move(L));
    return h;
  }
  return 0;
}

static kvbm_paged_layout descriptor(const Layout& L)
{
  kvbm_paged_layout d{};
  d.layer_base = L.dev_layer_base;
  d.block_stride = L.block_stride;
  d.outer_stride = L.outer_stride;
  d.region_bytes = static_cast<uint32_t>(L.region);
  d.num_layers = static_cast<uint32_t>(L.cfg.num_layers);
  d.outer_dim = static_cast<uint32_t>(L.cfg.outer_dim);
  d.num_blocks = static_cast<uint32_t>(L.cfg.num_blocks);
  return d;
}

// memcpy.rs:98-165
// executor/memcpy.rs:30-165.  The reference copies chunk after chunk on the calling thread; here the chunk list is
// resolved (and fully validated) first and large requests are split over host threads -- destination blocks are
// unique (validate_block_transfer), so the pieces are disjoint.  Still synchronous: returns when every byte is written.
struct HostCopy {
  void* dst;
  const void* src;
  size_t bytes;
};

static unsigned memcpy_threads()
{
  static const unsigned n = [] {
    if (const char* e = std::getenv("KVBM_MEMCPY_THREADS")) {
      const long v = std::atol(e);
      if (v >= 1) return static_cast<unsigned>(std::min<long>(v, 256));
    }
    const unsigned hw = std::thread::hardware_concurrency();
    return std::max(1u, std::min(hw ? hw : 1u, 32u));   // memory-bound: more threads than memory channels buys nothing
  }();
  return n;
}

static void run_host_copies(const std::vector<HostCopy>& cs)
{
  size_t total = 0;
  for (const HostCopy& c : cs) total += c.bytes;
  const unsigned want = memcpy_threads();
  constexpr size_t kParallelFrom = 8u << 20;   // below this the thread start-up costs more than it saves
  if (want <= 1 || total < kParallelFrom || cs.size() < 2) {
    for (const HostCopy& c : cs) std::memcpy(c.dst, c.src, c.bytes);
    return;
  }
  const unsigned T = static_cast<unsigned>(std::min<size_t>(want, cs.size()));
  auto work = [&](unsigned t) {
    const size_t lo = cs.size() * t / T, hi = cs.size() * (t + 1) / T;
    for (size_t i = lo; i < hi; ++i) std::memcpy(cs[i].dst, cs[i].src, cs[i].bytes);
  };
  std::vector<std::thread> th;
  th.reserve(T - 1);
  for (unsigned t = 1; t < T; ++t) th.emplace_back(work, t);
  work(0);
  for (auto& x : th) x.join();
}

static int host_memcpy_transfer(const Layout& S, const Layout& D, const size_t* sid, const size_t* did, size_t n,
                                bool has_range, size_t lb, size_t le)
{
  const bool full = !has_range || (lb == 0 && le == S.cfg.num_layers);
  std::string why;
  std::vector<HostCopy> cs;
  if (full && S.fully_contiguous && D.fully_contiguous) {  // can_use_whole_block_transfer, transfer/mod.rs:150-173
    const size_t bytes = bytes_per_block(S.cfg);
    cs.reserve(n);
    for (size_t i = 0; i < n; ++i) {
      uintptr_t s, d;
      int rc;
      if ((rc = S.memory_region(sid[i], 0, 0, &s, nullptr, &why))) return fail(rc, why);
      if ((rc = D.memory_region(did[i], 0, 0, &d, nullptr, &why))) return fail(rc, why);
      cs.push_back({reinterpret_cast<void*>(d), reinterpret_cast<const void*>(s), bytes});
    }
    run_host_copies(cs);
    return KVBM_OK;
  }
  cs.reserve(n * (le - lb) * S.cfg.outer_dim);
  for (size_t i = 0; i < n; ++i)
    for (size_t l = lb; l < le; ++l)
      for (size_t o = 0; o < S.cfg.outer_dim; ++o) {
        uintptr_t s, d;
        size_t ss, ds;
        int rc;
        if ((rc = S.memory_region(sid[i], l, o, &s, &ss, &why))) return fail(rc, why);
        if ((rc = D.memory_region(did[i], l, o, &d, &ds, &why))) return fail(rc, why);
        if (ss != ds)
          return fail(KVBM_ERR_INCOMPATIBLE, "Memory region size mismatch at block=(" + std::to_string(sid[i]) + "," + std::to_string(did[i]) +
                                                 "), layer=" + std::to_string(l) + ", outer=" + std::to_string(o) + ": src=" + std::to_string(ss) +
                                                 ", dst=" + std::to_string(ds));
        cs.push_back({reinterpret_cast<void*>(d), reinterpret_cast<const void*>(s), ss});
      }
  run_host_copies(cs);
  return KVBM_OK;
}

// (Re)size one slot's resources.  cudaMalloc / cudaHostAlloc / cudaMemset synchronise the device, which would
// deadlock against a gated (layer-streaming) transfer that is still spinning on its ready flags -- so every slot
// is provisioned when the manager is created and this only runs again for unusually large requests.
static int ensure_slot(Slot& sl, size_t ids_needed, size_t ws_needed)
{
  if (!sl.ev) CU(cudaEventCreateWithFlags(&sl.ev, cudaEventDisableTiming));
  if (!sl.host_flag) {
    CU(cudaHostAlloc(reinterpret_cast<void**>(&sl.host_flag), 64, cudaHostAllocMapped | cudaHostAllocPortable));
    *sl.host_flag = 0;
    sl.owns_flag = true;
  }
  if (sl.cap < ids_needed) {
    if (sl.owns_ids) {
      if (sl.pinned_ids) cudaFreeHost(sl.pinned_ids);
      if (sl.dev_ids) cudaFree(sl.dev_ids);
    }
    sl.pinned_ids = nullptr;
    sl.dev_ids = nullptr;
    sl.cap = 0;
    size_t cap = 4096;
    while (cap < ids_needed) cap *= 2;
    CU(cudaHostAlloc(reinterpret_cast<void**>(&sl.pinned_ids), cap * sizeof(int32_t), cudaHostAllocPortable));
    sl.owns_ids = true;
    CU(cudaMalloc(reinterpret_cast<void**>(&sl.dev_ids), cap * sizeof(int32_t)));
    sl.cap = cap;
  }
  if (sl.ws_cap < ws_needed) {
    if (sl.owns_ws && sl.dev_ws) cudaFree(sl.dev_ws);
    sl.dev_ws = nullptr;
    sl.ws_cap = 0;
    size_t cap = 512;
    while (cap < ws_needed) cap *= 2;
    CU(cudaMalloc(reinterpret_cast<void**>(&sl.dev_ws), cap * sizeof(uint32_t)));
    sl.owns_ws = true;
    CU(cudaMemset(sl.dev_ws, 0, cap * sizeof(uint32_t)));
    sl.ws_cap = cap;
  }
  return KVBM_OK;
}

// Carve every slot's default share out of two arenas (called once, device current).
static int provision_slots(kvbm_transfer_manager* m)
{
  const size_t pin_per = kArenaIds * sizeof(int32_t) + 64;                       // ids + flag word (own cache line)
  const size_t dev_per = kArenaIds * sizeof(int32_t) + kArenaWs * sizeof(uint32_t);
  CU(cudaHostAlloc(reinterpret_cast<void**>(&m->pinned_arena), pin_per * kSlots, cudaHostAllocMapped | cudaHostAllocPortable));
  CU(cudaMalloc(reinterpret_cast<void**>(&m->dev_arena), dev_per * kSlots));
  CU(cudaMemset(m->dev_arena, 0, dev_per * kSlots));
  std::memset(m->pinned_arena, 0, pin_per * kSlots);
  for (int i = 0; i < kSlots; ++i) {
    Slot& sl = m->slots[i];
    uint8_t* hp = m->pinned_arena + pin_per * i;
    uint8_t* dp = m->dev_arena + dev_per * i;
    sl.pinned_ids = reinterpret_cast<int32_t*>(hp);
    sl.host_flag = reinterpret_cast<uint32_t*>(hp + kArenaIds * sizeof(int32_t));
    sl.dev_ids = reinterpret_cast<int32_t*>(dp);
    sl.dev_ws = reinterpret_cast<uint32_t*>(dp + kArenaIds * sizeof(int32_t));
    sl.cap = kArenaIds;
    sl.ws_cap = kArenaWs;
    CU(cudaEventCreateWithFlags(&sl.ev, cudaEventDisableTiming));
  }
  return KVBM_OK;
}

// Acquire a slot whose previous transfer has completed (waits for the oldest if all are busy).
static int acquire_slot(kvbm_transfer_manager* m, size_t ids_needed, size_t ws_needed, Slot** out, uint64_t* seq)
{
  const uint64_t s = m->next_seq++;
  Slot& sl = m->slots[(s - 1) % kSlots];
  if (sl.in_flight) {
    CU(cudaEventSynchronize(sl.ev));
    sl.in_flight = false;
  }
  int rc = ensure_slot(sl, ids_needed, ws_needed);
  if (rc) return rc;
  // the previous owner has completed: clear its completion word (an abort marker must not be mistaken for ours) BEFORE
  // the new owner is published
  __atomic_store_n(sl.host_flag, 0u, __ATOMIC_RELAXED);
  sl.seq.store(s, std::memory_order_release);
  *out = &sl;
  *seq = s;
  return KVBM_OK;
}

// The block tables of one launch on `stream`, optionally ordered after `wait_ev`: acquire a slot, narrow list k (lens[k] ids) to
// int32 right after list k - 1 in its pinned staging (a null list leaves its run unwritten) and upload all of them with one async
// copy (no host sync; the reference blocks on pointers_transfered_event.synchronize(), cuda.rs:324).
// units (a batch's unit table, num_units 16 B records) travels in the same copy, behind the ids at units_at(total ids).
static size_t units_at(size_t total_ids) { return (total_ids + 3) & ~size_t{3}; }  // in int32 entries: 16 B aligned in the slot

static int stage_ids(kvbm_transfer_manager* m, const size_t* const* lists, const size_t* lens, size_t num_lists, size_t ws_needed,
                     cudaStream_t stream, cudaEvent_t wait_ev, Slot** out, uint64_t* seq, const kvbm_repage_unit* units = nullptr,
                     size_t num_units = 0)
{
  size_t total = 0;
  for (size_t k = 0; k < num_lists; ++k) total += lens[k];
  const size_t words = num_units ? units_at(total) + num_units * (sizeof(kvbm_repage_unit) / sizeof(int32_t)) : total;
  int rc = acquire_slot(m, words, ws_needed, out, seq);
  if (rc) return rc;
  Slot* sl = *out;
  if (wait_ev) CU(cudaStreamWaitEvent(stream, wait_ev, 0));
  for (size_t k = 0, at = 0; k < num_lists; at += lens[k++])
    if (lists[k])
      for (size_t i = 0; i < lens[k]; ++i) sl->pinned_ids[at + i] = static_cast<int32_t>(lists[k][i]);
  if (num_units) std::memcpy(sl->pinned_ids + units_at(total), units, num_units * sizeof(kvbm_repage_unit));
  CU(cudaMemcpyAsync(sl->dev_ids, sl->pinned_ids, words * sizeof(int32_t), cudaMemcpyHostToDevice, stream));
  m->h2d_bytes += words * sizeof(int32_t);
  return KVBM_OK;
}

// Lists of n ids each: list k at k * n.  A fan-out's lists fit on the stack; a gather may name any number of sources.
static int stage_ids(kvbm_transfer_manager* m, const size_t* const* lists, size_t num_lists, size_t n, size_t ws_needed,
                     cudaStream_t stream, cudaEvent_t wait_ev, Slot** out, uint64_t* seq)
{
  size_t stack[2 * KVBM_MAX_DESTINATIONS + 1];
  std::vector<size_t> heap;
  size_t* lens = stack;
  if (num_lists > sizeof(stack) / sizeof(stack[0])) {
    heap.resize(num_lists);
    lens = heap.data();
  }
  for (size_t k = 0; k < num_lists; ++k) lens[k] = n;
  return stage_ids(m, lists, lens, num_lists, ws_needed, stream, wait_ev, out, seq);
}

// After the launch: the slot stays busy until its event, and the launch's payload is counted.
static int finish_slot(kvbm_transfer_manager* m, Slot* sl, cudaStream_t stream, uint64_t bytes)
{
  CU(cudaEventRecord(sl->ev, stream));
  sl->in_flight = true;
  m->bytes_moved += bytes;
  return KVBM_OK;
}

// heads: a head-window transfer, whose regions differ when the head counts do; the head rows (head_dim elements) must match
// instead.  Both configs then carry num_heads dividing inner_dim (checked by the caller).  staged: a staged gather's pair, whose
// layer windows map layers between pools of different layer counts.
static int check_compat(const Layout& S, const Layout& D, int cast, bool heads = false, bool staged = false)
{
  if (!staged && S.cfg.num_layers != D.cfg.num_layers)  // executor/cuda.rs:52-58, memcpy.rs:49-55
    return fail(KVBM_ERR_INCOMPATIBLE, "Layouts have incompatible layer counts: src=" + std::to_string(S.cfg.num_layers) +
                                           ", dst=" + std::to_string(D.cfg.num_layers));
  if (S.cfg.outer_dim != D.cfg.outer_dim)  // cuda.rs:60-66
    return fail(KVBM_ERR_INCOMPATIBLE, "Layouts have incompatible outer dimensions: src=" + std::to_string(S.cfg.outer_dim) +
                                           ", dst=" + std::to_string(D.cfg.outer_dim));
  const size_t num = cast == KVBM_CAST_FP8E4M3_TO_BF16 ? 2 : 1, den = cast == KVBM_CAST_BF16_TO_FP8E4M3 ? 2 : 1;
  if (heads) {
    const size_t s_row = S.cfg.inner_dim / S.cfg.num_heads * S.cfg.dtype_width_bytes, d_row = D.cfg.inner_dim / D.cfg.num_heads * D.cfg.dtype_width_bytes;
    if (s_row * num != d_row * den)
      return fail(KVBM_ERR_INCOMPATIBLE, "Head row size mismatch: src=" + std::to_string(s_row) + ", dst=" + std::to_string(d_row));
  } else if (S.region * num != D.region * den)
    return fail(KVBM_ERR_INCOMPATIBLE, "Memory region size mismatch: src=" + std::to_string(S.region) + ", dst=" + std::to_string(D.region));
  if (cast == KVBM_CAST_FP8E4M3_TO_BF16 && (S.cfg.dtype_width_bytes != 1 || D.cfg.dtype_width_bytes != 2))
    return fail(KVBM_ERR_INCOMPATIBLE, "fp8->bf16 cast needs dtype widths 1 -> 2");
  if (cast == KVBM_CAST_BF16_TO_FP8E4M3 && (S.cfg.dtype_width_bytes != 2 || D.cfg.dtype_width_bytes != 1))
    return fail(KVBM_ERR_INCOMPATIBLE, "bf16->fp8 cast needs dtype widths 2 -> 1");
  return KVBM_OK;
}

// One block-table kernel launch (execute_cuda_transfer, executor/cuda.rs:39-156) on `stream`, optionally ordered after
// `wait_ev`.  The manager mutex is held by the caller.
static int launch_cuda(kvbm_transfer_manager* m, Layout* S, Layout* const* D, int nd, const size_t* const* src_ids,
                       const size_t* const* dst_ids, size_t n, bool replicate, size_t lb, size_t le,
                       const kvbm_transfer_options& o, cudaStream_t stream, cudaEvent_t wait_ev, Slot** slot_out, uint64_t* seq_out)
{
  // block tables: replicate = [src, dst 0, dst 1, ...], otherwise [src 0, dst 0, src 1, dst 1, ...]
  const size_t* lists[2 * KVBM_MAX_DESTINATIONS];
  size_t k = 0;
  if (replicate) lists[k++] = src_ids[0];
  for (int d = 0; d < nd; ++d) {
    if (!replicate) lists[k++] = src_ids[d];
    lists[k++] = dst_ids[d];
  }
  Slot* sl;
  uint64_t seq;
  int rc = stage_ids(m, lists, k, n, S->cfg.num_layers + 4, stream, wait_ev, &sl, &seq);
  if (rc) return rc;

  kvbm_paged_layout sdesc = descriptor(*S);
  kvbm_paged_dst dd[KVBM_MAX_DESTINATIONS] = {};
  uint64_t bytes = 0;
  for (int d = 0; d < nd; ++d) {
    dd[d].layout = descriptor(*D[d]);
    dd[d].src_block_ids = sl->dev_ids + (replicate ? 0 : 2 * d) * n;
    dd[d].dst_block_ids = sl->dev_ids + (replicate ? 1 + d : 2 * d + 1) * n;
    dd[d].done_flag = o.per_dst_done_flags ? o.per_dst_done_flags[d] : ((d == 0) ? o.done_flag : nullptr);
    dd[d].layer_done_flags = o.per_dst_layer_done_flags ? o.per_dst_layer_done_flags[d] : ((d == 0) ? o.layer_done_flags : nullptr);
    bytes += n * (le - lb) * S->cfg.outer_dim * D[d]->region;
  }
  kvbm_paged_copy_opts ko{};
  ko.epoch = o.epoch;
  ko.layer_ready_flags = o.layer_ready_flags;
  ko.sync_workspace = sl->dev_ws;
  ko.max_ctas = o.max_ctas;
  ko.gate_timeout_ms = o.gate_timeout_ms;
  ko.gate_mode = o.gate_mode;
  ko.multicast = o.multicast;
  ko.completion_flag = sl->host_flag;
  ko.completion_value = static_cast<uint32_t>(seq);
  ko.cast_scales = o.cast_scales;
  cudaError_t e = kvbm_kernels_paged_copy_v2(&sdesc, dd, nd, static_cast<int>(n), static_cast<int>(lb), static_cast<int>(le), o.cast_mode, &ko, stream);
  if (e != cudaSuccess) return fail_cuda(e, "kvbm_kernels_paged_copy_v2");
  if ((rc = finish_slot(m, sl, stream, bytes))) return rc;
  *slot_out = sl;
  *seq_out = seq;
  return KVBM_OK;
}

// A request as resolve() (or the re-paging checks) validated it: its layouts and effective formats (the options override a
// layout's own), whether it takes the permuting launch and with which head window (the whole source unless the request names
// one), the layer range, the strategy plan and a two-hop plan's bounce layout.  `empty`: nothing to move (no blocks or an empty
// layer range); nothing after the layer range is resolved then.
struct Transfer {
  Layout* S = nullptr;
  Layout* D[KVBM_MAX_DESTINATIONS] = {};
  Layout* B = nullptr;
  int src_kv = KVBM_KV_UNKNOWN, dst_kv = KVBM_KV_UNKNOWN;  // dst_kv: of D[0]
  bool permute = false;
  kvbm_head_window window{};
  size_t lb = 0, le = 0;
  kvbm_transfer_plan plan{};
  bool empty = false;
};

// The gate of a streamed launch: window j reads source e[j].window.src_rank, so it waits for that source's flags; the options'
// epoch, gate mode, timeout, CTA cap and done flag; the slot's workspace and completion word.
static kvbm_permute_stream layer_stream(const kvbm_layer_stream& ls, const Transfer* e, size_t nw, const kvbm_transfer_options& o,
                                        const Slot& sl, uint64_t seq)
{
  kvbm_permute_stream st{};
  for (size_t j = 0; j < nw; ++j) st.layer_ready_flags[j] = ls.src_layer_ready_flags[e[j].window.src_rank];
  st.layer_done_flags = ls.layer_done_flags;
  st.done_flag = o.done_flag;
  st.epoch = o.epoch;
  st.sync_workspace = sl.dev_ws;
  st.completion_flag = sl.host_flag;
  st.completion_value = static_cast<uint32_t>(seq);
  st.gate_mode = o.gate_mode;
  st.gate_timeout_ms = o.gate_timeout_ms;
  st.max_ctas = o.max_ctas;
  return st;
}

static int checked(cudaError_t e, const char* what) { return e == cudaSuccess ? KVBM_OK : fail_cuda(e, what); }

// The launch every layout-transforming hand-off ends with, on `stream`.  One slot takes the block tables [source 0 ..
// num_srcs - 1 (n_src ids each), destination (n_dst ids)] and, with ls, a workspace over the destination's layers.  Window j
// becomes the kvbm_permute_source of e[j]'s source and head window, reading table e[j].window.src_rank; the destination's side
// is e[0]'s; with ls, the gate.  `launch(sources, destination, gate or null, slot, seq)` makes the kernel call and returns its
// code.  Then the slot counts `bytes`, *seq_out gets the launch's sequence number and *out the notification: 0 on a caller
// stream, whose caller manages sync.  units: a batch's unit table, staged behind the tables at units_at(every id) of the slot.
template <class Launch>
static int launch_transform(kvbm_transfer_manager* m, const Transfer* e, size_t nw, size_t num_srcs, const size_t* const* src_ids,
                            size_t n_src, const size_t* dst_ids, size_t n_dst, const kvbm_layer_stream* ls, const kvbm_transfer_options& o,
                            cudaStream_t stream, uint64_t bytes, uint64_t* seq_out, kvbm_notification* out, Launch&& launch,
                            const kvbm_repage_unit* units = nullptr, size_t num_units = 0)
{
  // the tables' pointers and lengths fit on the stack for every request that names only the sources its windows read; a
  // gather may pass any number of sources
  const size_t k = num_srcs + 1;
  const size_t* stack_lists[KVBM_GATHER_MAX_SOURCES + 1];
  size_t stack_lens[KVBM_GATHER_MAX_SOURCES + 1];
  std::vector<const size_t*> heap_lists;
  std::vector<size_t> heap_lens;
  const size_t** lists = stack_lists;
  size_t* lens = stack_lens;
  if (k > KVBM_GATHER_MAX_SOURCES + 1) {
    heap_lists.resize(k);
    heap_lens.resize(k);
    lists = heap_lists.data();
    lens = heap_lens.data();
  }
  std::copy(src_ids, src_ids + num_srcs, lists);
  std::fill(lens, lens + num_srcs, n_src);
  lists[num_srcs] = dst_ids;
  lens[num_srcs] = n_dst;
  const Layout& D = *e[0].D[0];
  Slot* sl;
  uint64_t seq;
  int rc = stage_ids(m, lists, lens, k, ls ? D.cfg.num_layers + 4 : 4, stream, nullptr, &sl, &seq, units, num_units);
  if (rc) return rc;
  const kvbm_permute_side kd{descriptor(D), sl->dev_ids + num_srcs * n_src, e[0].dst_kv};
  kvbm_permute_source ks[KVBM_GATHER_MAX_SOURCES] = {};
  for (size_t j = 0; j < nw; ++j) {
    const kvbm_head_window& w = e[j].window;
    ks[j] = kvbm_permute_source{{descriptor(*e[j].S), sl->dev_ids + w.src_rank * n_src, e[j].src_kv}, static_cast<uint32_t>(e[j].S->cfg.num_heads),
                                static_cast<uint32_t>(w.src_head_begin), static_cast<uint32_t>(w.dst_head_begin),
                                static_cast<uint32_t>(w.head_count)};
  }
  kvbm_permute_stream st{};
  if (ls) st = layer_stream(*ls, e, nw, o, *sl, seq);
  if ((rc = launch(ks, kd, ls ? &st : nullptr, *sl, seq))) return rc;
  if ((rc = finish_slot(m, sl, stream, bytes))) return rc;
  if (seq_out) *seq_out = seq;
  if (out) *out = o.use_caller_stream ? 0 : seq;
  return KVBM_OK;
}

// What a layout-transforming launch moves: `units` (blocks or tokens) x each window's layers inside [lb, le) (layers[j]'s layer
// window, or every layer) x the outer dimension x its heads x `head_bytes`, a destination head's bytes per unit.
static uint64_t transform_bytes(const Transfer* e, size_t nw, const kvbm_shard_window* layers, size_t lb, size_t le, uint64_t units,
                                uint64_t head_bytes)
{
  uint64_t bytes = 0;
  for (size_t j = 0; j < nw; ++j) {
    size_t from = lb, to = le;
    if (layers) {
      from = std::max(from, layers[j].dst_layer_begin);
      to = std::min(to, layers[j].dst_layer_begin + layers[j].layer_count);
    }
    if (to > from) bytes += units * (to - from) * e[0].D[0]->cfg.outer_dim * e[j].window.head_count * head_bytes;
  }
  return bytes;
}

// The kernel sources of a launch: window j's gather source with the layer window of layers[j], or without layers the identity
// window over the destination's nl layers (an unstaged request, whose sources check_compat gave the destination's layer count).
static void stage_sources(const kvbm_permute_source* ks, const kvbm_shard_window* layers, size_t nw, size_t nl, kvbm_stage_source* ss)
{
  for (size_t j = 0; j < nw; ++j)
    ss[j] = layers ? kvbm_stage_source{ks[j], static_cast<uint32_t>(layers[j].src_layer_begin), static_cast<uint32_t>(layers[j].dst_layer_begin),
                                       static_cast<uint32_t>(layers[j].layer_count)}
                   : kvbm_stage_source{ks[j], 0, 0, static_cast<uint32_t>(nl)};
}

// The layout-transforming transfer: what select_transform_kernel's result would drive if the reference ran it inside
// execute_transfer (it rejects the pair instead, transfer/mod.rs:128-147).  One permuting launch moves every entry's head window
// from source e[j].window.src_rank into e[0].D over e[0]'s layer range, with the transfer's fp8 <-> bf16 cast fused in:
// kvbm_kernels_paged_permute_heads_scaled for one unstaged, unstreamed window (any head count), else
// kvbm_kernels_paged_stage_gather, or its streamed form with ls (gated on every window's source flags).  Every source list and
// the destination's hold n ids; the completion word is written by a trailing signal kernel.
// layers: a staged gather, window j with the layer window of layers[j]; without, every window is one stage over the
// destination's layers.  Each window's bytes count over its layers inside the layer range.
// *seq_out: the launch's sequence number; *out: the notification, as launch_transform sets them (either may be null).
static int launch_permute(kvbm_transfer_manager* m, const Transfer* e, size_t nw, size_t num_srcs, const size_t* const* src_ids,
                          const size_t* dst_ids, size_t n, const kvbm_transfer_options& o, cudaStream_t stream, uint64_t* seq_out,
                          kvbm_notification* out = nullptr, const kvbm_layer_stream* ls = nullptr, const kvbm_shard_window* layers = nullptr)
{
  const Layout *S0 = e[0].S, *D = e[0].D[0];
  const uint64_t bytes = transform_bytes(e, nw, layers, e[0].lb, e[0].le, n, D->region / D->cfg.num_heads);
  const uint32_t dnh = static_cast<uint32_t>(D->cfg.num_heads), page = static_cast<uint32_t>(S0->cfg.page_size);
  const uint32_t row = static_cast<uint32_t>(S0->cfg.inner_dim / S0->cfg.num_heads * S0->cfg.dtype_width_bytes);
  const int nb = static_cast<int>(n), lb = static_cast<int>(e[0].lb), le = static_cast<int>(e[0].le), k = static_cast<int>(nw);
  auto launch = [&](const kvbm_permute_source* ks, const kvbm_permute_side& kd, const kvbm_permute_stream* st, const Slot& sl, uint64_t seq) {
    const uint32_t value = static_cast<uint32_t>(seq);
    if (nw == 1 && !layers && !st)
      return checked(kvbm_kernels_paged_permute_heads_scaled(&ks[0].side, &kd, nb, lb, le, ks[0].num_heads, ks[0].src_head_begin, dnh,
                                                             ks[0].dst_head_begin, ks[0].head_count, page, row, o.cast_mode, o.cast_scales,
                                                             o.done_flag, o.epoch, sl.host_flag, value, stream),
                     "kvbm_kernels_paged_permute_heads_scaled");
    kvbm_stage_source ss[KVBM_GATHER_MAX_SOURCES] = {};
    stage_sources(ks, layers, nw, D->cfg.num_layers, ss);
    if (st)
      return checked(kvbm_kernels_paged_stage_gather_streamed(ss, k, &kd, dnh, nb, lb, le, page, row, o.cast_mode, o.cast_scales, st, stream),
                     "kvbm_kernels_paged_stage_gather_streamed");
    return checked(kvbm_kernels_paged_stage_gather(ss, k, &kd, dnh, nb, lb, le, page, row, o.cast_mode, o.cast_scales, o.done_flag, o.epoch,
                                                   sl.host_flag, value, stream),
                   "kvbm_kernels_paged_stage_gather");
  };
  return launch_transform(m, e, nw, num_srcs, src_ids, n, dst_ids, n, ls, o, stream, bytes, seq_out, out, launch);
}

// Whether kernels on the manager's device can use p: its own device memory, pinned host memory mapped into its address space,
// or, with `peers`, memory of a device it has peer access to (enabled through kvbm_manager_enable_peer_access, or by an IPC
// mapping this manager opened).  Pageable host memory and any other device's memory cannot be.
static bool reachable(const kvbm_transfer_manager* m, const void* p, bool peers)
{
  cudaPointerAttributes a{};
  if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
    (void)cudaGetLastError();
    return false;
  }
  if (a.type == cudaMemoryTypeHost) return a.devicePointer == p;
  return a.type == cudaMemoryTypeDevice && (a.device == m->device || (peers && m->peers.count(a.device) != 0));
}

// The cast kernels read the scales on the manager's device, never through a peer.
static int check_cast_scales(kvbm_transfer_manager* m, const float* p)
{
  if (!reachable(m, p, false))
    return fail(KVBM_ERR, "cast_scales must be device memory of device " + std::to_string(m->device) +
                              " or pinned host memory mapped into it (a pageable or another device's pointer cannot be read by the cast)");
  return KVBM_OK;
}

// The shape of a streamed request's flags, before anything else is checked: one ready-flag array per source, none null.
static int check_layer_stream_shape(const kvbm_layer_stream* ls, size_t num_srcs)
{
  if (!ls || !ls->src_layer_ready_flags) return fail(KVBM_ERR, "a streamed transfer needs a kvbm_layer_stream with ready flags");
  if (ls->num_srcs != num_srcs)
    return fail(KVBM_ERR_LENGTH_MISMATCH, "the layer stream names " + std::to_string(ls->num_srcs) + " sources' ready flags, the request has " +
                                              std::to_string(num_srcs) + " sources");
  for (size_t s = 0; s < num_srcs; ++s)
    if (!ls->src_layer_ready_flags[s]) return fail(KVBM_ERR, "source " + std::to_string(s) + " has no layer ready flags");
  return KVBM_OK;
}

// The flags of a streamed request are polled and written by the kernels on the manager's device, which may reach them through
// a peer: the ready flags of every window's source (e[j].window.src_rank) and the layer done flags.
static int check_layer_stream_flags(kvbm_transfer_manager* m, const kvbm_layer_stream& ls, const Transfer* e, size_t nw)
{
  for (size_t j = 0; j < nw; ++j) {
    const size_t r = e[j].window.src_rank;
    if (!reachable(m, ls.src_layer_ready_flags[r], true))
      return fail(KVBM_ERR, "the layer ready flags of source " + std::to_string(r) + " are not reachable from device " +
                                std::to_string(m->device) + " (its own memory, a device it has peer access to, or mapped pinned host memory)");
  }
  if (ls.layer_done_flags && !reachable(m, ls.layer_done_flags, true))
    return fail(KVBM_ERR, "the layer done flags are not reachable from device " + std::to_string(m->device) +
                              " (its own memory, a device it has peer access to, or mapped pinned host memory)");
  return KVBM_OK;
}

static bool cuda_strategy(int s) { return s == KVBM_STRATEGY_CUDA_ASYNC_H2D || s == KVBM_STRATEGY_CUDA_ASYNC_D2H || s == KVBM_STRATEGY_CUDA_ASYNC_D2D; }

// The stream of a CUDA strategy: the caller's, or round-robin from the pool (cuda.rs:82-90: D2H pool for D2H, H2D pool otherwise).
static cudaStream_t pick_stream(kvbm_transfer_manager* m, int strategy, const kvbm_transfer_options& o)
{
  if (o.use_caller_stream) return o.cuda_stream;
  return strategy == KVBM_STRATEGY_CUDA_ASYNC_D2H ? m->d2h[m->rr_d2h++ % kStreams] : m->h2d[m->rr_h2d++ % kStreams];
}

// execute_two_hop_transfer (executor/mod.rs:477-571) with handle_buffered_transfer's two bounce groups (:357-416): the
// bounce blocks are split in two halves; chunk i goes src -> half (i & 1) -> dst.  The reference runs two tokio tasks
// that each await their hops; here both hops are stream work ordered by events, so chunk i+1's first hop overlaps chunk
// i's second hop and the host never blocks.  One bounce block = strictly sequential, like the reference (:526-548).
static int execute_two_hop(kvbm_transfer_manager* m, Layout* S, Layout* D, Layout* B, const size_t* src_ids, const size_t* dst_ids,
                           size_t n, const size_t* bounce_ids, size_t nb, size_t lb, size_t le, const kvbm_transfer_plan& plan,
                           const kvbm_transfer_options& o, kvbm_notification* out)
{
  cudaStream_t s1 = pick_stream(m, plan.first, o), s2 = pick_stream(m, plan.second, o);  // never the caller's: resolve() rejects it
  nb = std::min(nb, n);
  const size_t half = nb >= 2 ? nb / 2 : nb;
  const size_t group_begin[2] = {0, half};
  const size_t group_len[2] = {half, nb >= 2 ? nb - half : 0};
  const int groups = nb >= 2 ? 2 : 1;
  cudaEvent_t hop2_done[2] = {nullptr, nullptr};
  kvbm_transfer_options o1 = o, o2 = o;
  o1.done_flag = nullptr;        // completion signals belong to the hop that lands the bytes at the destination
  o1.per_dst_done_flags = nullptr;  // (layer streaming is rejected by check_strategy)
  uint64_t last = 0;
  size_t pos = 0;
  for (int c = 0; pos < n; ++c) {
    const int g = c % groups;
    const size_t cnt = std::min(group_len[g], n - pos);
    const size_t* bids = bounce_ids + group_begin[g];
    const size_t* sp = src_ids + pos;
    const size_t* dp = dst_ids + pos;
    Slot *a, *b;
    uint64_t sa, sb;
    Layout* Bp = B;
    int rc = launch_cuda(m, S, &Bp, 1, &sp, &bids, cnt, true, lb, le, o1, s1, hop2_done[g], &a, &sa);
    if (rc) return rc;
    Layout* Dp = D;
    kvbm_transfer_options o2c = o2;
    if (pos + cnt < n) {  // only the last chunk announces the whole transfer
      o2c.done_flag = nullptr;
      o2c.per_dst_done_flags = nullptr;
    }
    rc = launch_cuda(m, B, &Dp, 1, &bids, &dp, cnt, true, lb, le, o2c, s2, a->ev, &b, &sb);
    if (rc) return rc;
    hop2_done[g] = b->ev;
    last = sb;
    pos += cnt;
  }
  if (out) *out = last;
  return KVBM_OK;
}

// Checks that both the head-window block and the permuting path of resolve() make.  Each runs from both places because a
// request failing several checks reports the first one in the order the two blocks make them.
static int need_one_destination(int nd)
{
  return nd == 1 ? KVBM_OK : fail(KVBM_ERR_UNSUPPORTED, "a layout-transforming transfer takes one destination");
}
// LayoutConfig::validate_for_kv_block_layout (config.rs:118-126)
static int need_num_heads(const kvbm_layout_config& c)
{
  return c.num_heads ? KVBM_OK : fail(KVBM_ERR_CONFIG, "num_heads_required_for_kv_block_layout");
}
static int need_divisible_heads(const kvbm_layout_config& c)
{
  return c.inner_dim % c.num_heads ? fail(KVBM_ERR_CONFIG, "inner_dim_must_be_divisible_by_num_heads") : KVBM_OK;
}

// A head window (TP re-shard): both head counts known, the window inside both.
static int check_head_window(const Layout& S, const Layout& D, const kvbm_head_window& w, int nd)
{
  const kvbm_layout_config &sc = S.cfg, &dc = D.cfg;
  int rc;
  if ((rc = need_one_destination(nd)) || (rc = need_num_heads(sc)) || (rc = need_num_heads(dc)) || (rc = need_divisible_heads(sc)) ||
      (rc = need_divisible_heads(dc)))
    return rc;
  if (w.src_head_begin > sc.num_heads || w.head_count > sc.num_heads - w.src_head_begin || w.dst_head_begin > dc.num_heads ||
      w.head_count > dc.num_heads - w.dst_head_begin)
    return fail(KVBM_ERR_RANGE, "Head window src " + std::to_string(w.src_head_begin) + "+" + std::to_string(w.head_count) + " of " +
                                    std::to_string(sc.num_heads) + " heads, dst " + std::to_string(w.dst_head_begin) + "+" +
                                    std::to_string(w.head_count) + " of " + std::to_string(dc.num_heads) + " heads is out of range");
  return KVBM_OK;
}

static int check_walk(const Layout& S, const Layout& D, int src_kv, int dst_kv, int cast_mode);

// The permuting launch on one (source, destination) pair: one destination, no layer streaming or multicast, and the geometry
// the head-row walk needs.  With the fused cast the dtype widths differ as check_compat requires (1 -> 2 or 2 -> 1).
static int check_permute(const Layout& S, const Layout& D, int src_kv, int dst_kv, bool window, int nd, const kvbm_transfer_options& o)
{
  int rc;
  if ((rc = need_one_destination(nd))) return rc;
  if (o.layer_ready_flags || o.layer_done_flags || o.per_dst_done_flags || o.per_dst_layer_done_flags || o.multicast)
    return fail(KVBM_ERR_UNSUPPORTED, "layer streaming / multicast are not available on a layout-transforming transfer");
  const kvbm_layout_config &sc = S.cfg, &dc = D.cfg;
  if ((rc = need_num_heads(sc)) || (rc = need_num_heads(dc))) return rc;
  if (window) {  // the head counts may differ; the heads themselves may not
    if (sc.page_size != dc.page_size || sc.inner_dim / sc.num_heads != dc.inner_dim / dc.num_heads ||
        (o.cast_mode == KVBM_CAST_NONE && sc.dtype_width_bytes != dc.dtype_width_bytes))
      return fail(KVBM_ERR_INCOMPATIBLE, "a head-window transfer needs equal head_dim, page_size and dtype on both sides");
  } else if (sc.num_heads != dc.num_heads || sc.page_size != dc.page_size || sc.inner_dim != dc.inner_dim ||
             (o.cast_mode == KVBM_CAST_NONE && sc.dtype_width_bytes != dc.dtype_width_bytes))
    return fail(KVBM_ERR_INCOMPATIBLE, "a layout transformation needs equal num_heads, page_size, inner_dim and dtype on both sides");
  if ((rc = need_divisible_heads(sc))) return rc;  // after the equality above, the source's inner_dim speaks for both
  return check_walk(S, D, src_kv, dst_kv, o.cast_mode);
}

// What the head-row walk needs of a (source, destination) pair whose head_dim and dtypes check_compat accepted: whole 16-byte
// rows (the fp8 row with a cast), a fully contiguous pool under a universal format, 16-byte aligned pools and strides.
static int check_walk(const Layout& S, const Layout& D, int src_kv, int dst_kv, int cast_mode)
{
  const kvbm_layout_config& sc = S.cfg;
  const size_t head_dim = sc.inner_dim / sc.num_heads;
  if (cast_mode != KVBM_CAST_NONE) {  // the walk splits the fp8 row (head_dim bytes) into 16 B vectors
    if (head_dim < 16 || head_dim > 65536 || (head_dim & 15))
      return fail(KVBM_ERR_UNSUPPORTED, "layout transformation with the fused cast: head_dim must be a multiple of 16 in 16..65536 (the fp8 row in whole "
                                        "16-byte vectors), got " + std::to_string(head_dim));
  } else {
    const size_t row = head_dim * sc.dtype_width_bytes;
    if (row < 16 || row > 65536 || (row & 15))
      return fail(KVBM_ERR_UNSUPPORTED, "layout transformation: head_dim * dtype width must be a multiple of 16 bytes in 16..65536, got " + std::to_string(row));
  }
  const bool s_uni = src_kv == KVBM_KV_UNIVERSAL_TP || src_kv == KVBM_KV_UNIVERSAL_PP;
  const bool d_uni = dst_kv == KVBM_KV_UNIVERSAL_TP || dst_kv == KVBM_KV_UNIVERSAL_PP;
  if ((s_uni && !S.fully_contiguous) || (d_uni && !D.fully_contiguous))
    return fail(KVBM_ERR_INCOMPATIBLE, "a universal KV block layout needs a fully contiguous pool");
  auto aligned16 = [](const Layout& L) {
    if ((L.block_stride | L.outer_stride) & 15) return false;
    for (uint64_t b : L.layer_base)
      if (b & 15) return false;
    return true;
  };
  if (!aligned16(S) || !aligned16(D)) return fail(KVBM_ERR_UNSUPPORTED, "layout transformation needs 16-byte aligned pools and strides");
  return KVBM_OK;
}

static int need_cuda_device(const kvbm_transfer_manager* m)
{
  return m->device < 0 ? fail(KVBM_ERR_CUDA, "this TransferManager was created without a CUDA device; CUDA strategies have no CPU fallback")
                       : KVBM_OK;
}

// The rejections of the strategy t->plan names, in the order its path makes them, and a two-hop plan's bounce layout.  A
// permuting transfer passes them only on a direct CUDA strategy.
static int check_strategy(kvbm_transfer_manager* m, int nd, const kvbm_transfer_options& o, Transfer* t)
{
  const kvbm_transfer_plan& p = t->plan;
  if (!p.two_hop && p.first == KVBM_STRATEGY_MEMCPY) {
    if (o.cast_mode != KVBM_CAST_NONE) return fail(KVBM_ERR_UNSUPPORTED, "the fused cast exists only on the CUDA strategies");
    if (t->permute) return fail(KVBM_ERR_UNSUPPORTED, "layout transformations exist only on the CUDA strategies");
    if (o.use_caller_stream) return fail(KVBM_ERR_UNSUPPORTED, "cuda_stream option is not supported for Memcpy strategy");  // executor/mod.rs:272-276
    return KVBM_OK;
  }
  if (p.two_hop ? !cuda_strategy(p.first) || !cuda_strategy(p.second) : !cuda_strategy(p.first))
    return fail(KVBM_ERR_UNSUPPORTED, p.two_hop ? "two-hop plans with a NIXL (disk / remote agent) leg are outside this library"
                                                : "NIXL strategies are outside this library (the NVLink peer path replaces them)");
  if (int rc = need_cuda_device(m)) return rc;
  if (!p.two_hop) return o.cast_scales ? check_cast_scales(m, o.cast_scales) : KVBM_OK;
  if (nd != 1) return fail(KVBM_ERR_UNSUPPORTED, "two-hop transfers take one destination");
  if (o.use_caller_stream) return fail(KVBM_ERR_UNSUPPORTED, "Two-hop transfers don't support caller-provided streams");  // executor/mod.rs:441
  if (o.cast_mode != KVBM_CAST_NONE) return fail(KVBM_ERR_UNSUPPORTED, "the fused cast is not available on two-hop transfers");
  if (t->permute) return fail(KVBM_ERR_UNSUPPORTED, "a layout transformation is not available on two-hop transfers");
  // each chunk's first hop would be a whole gated launch and its second hop would announce layers other chunks have not landed
  if (o.layer_ready_flags || o.layer_done_flags || o.per_dst_layer_done_flags)
    return fail(KVBM_ERR_UNSUPPORTED, "layer streaming is not available on two-hop transfers");
  if (!o.bounce_layout || !o.bounce_block_ids || o.num_bounce_blocks == 0)
    return fail(KVBM_ERR, "Two-hop transfers require a bounce buffer.");  // executor/mod.rs:514-519
  Layout* B = t->B = m->find(o.bounce_layout);
  if (!B) return fail(KVBM_ERR_HANDLE, "invalid bounce buffer handle");
  if (B->storage != p.bounce_location) return fail(KVBM_ERR, "Bounce buffer layout does not match bounce location.");  // :521-527
  int rc;
  if ((rc = check_compat(*t->S, *B, KVBM_CAST_NONE)) || (rc = check_compat(*B, *t->D[0], KVBM_CAST_NONE))) return rc;
  std::unordered_set<size_t> seen;
  for (size_t i = 0; i < o.num_bounce_blocks; ++i) {
    if (o.bounce_block_ids[i] >= B->cfg.num_blocks) return fail(KVBM_ERR_RANGE, "bounce block id out of range");
    if (!seen.insert(o.bounce_block_ids[i]).second) return fail(KVBM_ERR_DUPLICATE_DST, "duplicate bounce block id");
  }
  return KVBM_OK;
}

// The options' layer range over the layers of `c` (filled into *lb / *le) and enough fp8 KV-cache scales: one per (layer, outer)
// of those layers, for the fp8 side of a cast.  `c` is the pool whose layers the range counts: the destination's for a staged
// gather, the source's otherwise.
static int check_layer_range(const kvbm_layout_config& c, const kvbm_transfer_options& o, size_t* lb, size_t* le)
{
  *lb = 0;
  *le = c.num_layers;
  if (o.has_layer_range) {
    *lb = o.layer_begin;
    *le = o.layer_end;
    if (*lb > *le || *le > c.num_layers)
      return fail(KVBM_ERR_RANGE, "Layer range " + std::to_string(*lb) + ".." + std::to_string(*le) + " exceeds num_layers " +
                                      std::to_string(c.num_layers));
  }
  if (o.cast_scales) {
    if (o.cast_mode == KVBM_CAST_NONE) return fail(KVBM_ERR, "cast_scales need a cast_mode: they scale the fp8 side of a cast");
    const size_t need = c.num_layers * c.outer_dim;
    if (o.num_cast_scales < need)
      return fail(KVBM_ERR_RANGE, "cast_scales holds " + std::to_string(o.num_cast_scales) + " scales, the pools need num_layers * outer_dim = " +
                                      std::to_string(need));
  }
  return KVBM_OK;
}

// Validate one request and resolve it into *t; the caller holds m->mu.  `heads`: a head window that always takes the permuting
// launch (a gather's).  Without it the options' window applies, and one over every head of both sides is the transfer without a
// window.  A request that fails several checks reports the first in the order below.  staged: a staged gather's window, whose
// source may have other layers than the destination; the layer range and the cast scales are then the destination's.
static int resolve(kvbm_transfer_manager* m, kvbm_layout_handle src_h, int nd, const kvbm_layout_handle* dst_h,
                   const size_t* const* src_ids, const size_t* const* dst_ids, size_t n, const kvbm_transfer_options& o,
                   const kvbm_head_window* heads, Transfer* t, bool staged = false)
{
  if (nd < 1 || nd > KVBM_MAX_DESTINATIONS) return fail(KVBM_ERR, "number of destinations must be in 1..=8");
  Layout* S = t->S = m->find(src_h);
  if (!S) return fail(KVBM_ERR_HANDLE, "invalid source handle");
  if (S->unmapped) return fail(KVBM_ERR_UNSUPPORTED, "source layout is a descriptor of another process's host memory: not addressable from this process");
  const kvbm_head_window w = heads ? *heads : kvbm_head_window{0, o.src_head_begin, o.dst_head_begin, o.head_count};
  bool window = false;
  for (int d = 0; d < nd; ++d) {
    Layout* D = t->D[d] = m->find(dst_h[d]);
    if (!D) return fail(KVBM_ERR_HANDLE, "invalid destination handle");
    if (D->unmapped) return fail(KVBM_ERR_UNSUPPORTED, "destination layout is a descriptor of another process's host memory: not addressable from this process");
    int rc;
    if (w.head_count) {
      if ((rc = check_head_window(*S, *D, w, nd))) return rc;
      window = heads || !(w.src_head_begin == 0 && w.dst_head_begin == 0 && w.head_count == S->cfg.num_heads && w.head_count == D->cfg.num_heads);
    }
    if ((rc = check_compat(*S, *D, o.cast_mode, window, staged))) return rc;
    if (n && (!src_ids || !dst_ids || !src_ids[d] || !dst_ids[d])) return fail(KVBM_ERR, "null block id list");
    if ((rc = validate_block_transfer(src_ids[d], n, dst_ids[d], n, S->cfg.num_blocks, D->cfg.num_blocks, src_h == dst_h[d]))) return rc;
  }
  for (int d = 0; d < nd; ++d)  // select_strategy, strategy.rs:86-90
    if (S->remote && t->D[d]->remote) return fail(KVBM_ERR_UNSUPPORTED, "Both src and dst are remote - this is not supported.");
  // effective_src_layout / effective_dst_layout (executor/mod.rs:103-119): the option overrides the layout's own format.
  // The reference rejects every pair that needs a transformation (validate_layout_compatibility, transfer/mod.rs:128-147);
  // here the pairs select_transform_kernel names -- plus UniversalTP <-> UniversalPP, its TODO -- run as ONE permuting launch.
  const int src_kv = t->src_kv = o.src_kv_layout ? o.src_kv_layout : S->kv_block_layout;
  for (int d = 0; d < nd; ++d) {
    const int dst_kv = o.dst_kv_layout ? o.dst_kv_layout : t->D[d]->kv_block_layout;
    int tk = select_transform_kernel(src_kv, dst_kv);
    if (tk == KVBM_TRANSFORM_UNSUPPORTED && (src_kv == KVBM_KV_UNIVERSAL_TP || src_kv == KVBM_KV_UNIVERSAL_PP) &&
        (dst_kv == KVBM_KV_UNIVERSAL_TP || dst_kv == KVBM_KV_UNIVERSAL_PP))
      tk = KVBM_TRANSFORM_UNIVERSAL_TO_UNIVERSAL;
    // a head window walks heads by the formats' strides, so both formats must be named ones
    if (tk == KVBM_TRANSFORM_UNSUPPORTED || (window && (!kv_known(src_kv) || !kv_known(dst_kv))))
      return fail(KVBM_ERR_UNSUPPORTED, std::string("Layout transformation not supported: src=") + kv_name(src_kv) + ", dst=" + kv_name(dst_kv));
    // a head window takes the permuting launch even between equal formats; more than one destination never gets past here
    t->permute = tk != KVBM_TRANSFORM_NONE || window;
    if (t->permute) {
      int rc = check_permute(*S, *t->D[d], src_kv, dst_kv, window, nd, o);
      if (rc) return rc;
    }
  }
  t->dst_kv = o.dst_kv_layout ? o.dst_kv_layout : t->D[0]->kv_block_layout;
  t->window = window ? w : kvbm_head_window{0, 0, 0, S->cfg.num_heads};  // a plain transform is the window over every head
  if (int rc = check_layer_range(staged ? t->D[0]->cfg : S->cfg, o, &t->lb, &t->le)) return rc;
  t->empty = n == 0 || t->lb == t->le;
  if (t->empty) return KVBM_OK;

  // select_strategy (strategy.rs:78-108): every layout handled here is local or peer-mapped
  for (int d = 0; d < nd; ++d) {
    const Layout& D = *t->D[d];
    kvbm_transfer_plan p{};
    int rc = select_direct_strategy(S->storage, D.storage, &m->caps, &p);
    if (rc) return rc;
    // strategy.rs:222-233,245-278: a device pool of ANOTHER GPU is "remote"; without GPU RDMA it is reached through
    // pinned host memory: TwoHop { CudaAsyncD2H, Pinned, CudaAsyncH2D }
    if (!p.two_hop && p.first == KVBM_STRATEGY_CUDA_ASYNC_D2D && !m->caps.allow_gpu_rdma &&
        (S->device_id != D.device_id || S->remote != D.remote))
      p = kvbm_transfer_plan{1, KVBM_STRATEGY_CUDA_ASYNC_D2H, KVBM_STORAGE_PINNED, KVBM_STRATEGY_CUDA_ASYNC_H2D};
    if (d && (p.first != t->plan.first || p.two_hop != t->plan.two_hop)) return fail(KVBM_ERR_UNSUPPORTED, "destinations need different strategies");
    t->plan = p;
  }
  return check_strategy(m, nd, o, t);
}

// execute_transfer / execute_fanout: one of four paths after validation -- two-hop, Memcpy, the permuting launch or the paged copy.
static int execute(kvbm_transfer_manager* m, kvbm_layout_handle src_h, int nd, const kvbm_layout_handle* dst_h,
                   const size_t* const* src_ids, const size_t* const* dst_ids, size_t n, bool replicate,
                   const kvbm_transfer_options* opts_in, kvbm_notification* out)
{
  kvbm_transfer_options o{};
  if (opts_in) o = *opts_in;
  if (out) *out = 0;
  std::lock_guard<std::mutex> lk(m->mu);
  Transfer t;
  int rc = resolve(m, src_h, nd, dst_h, src_ids, dst_ids, n, o, nullptr, &t);
  if (rc || t.empty) return rc;
  if (t.plan.two_hop) {
    DeviceGuard g(m->device);
    return execute_two_hop(m, t.S, t.D[0], t.B, src_ids[0], dst_ids[0], n, o.bounce_block_ids, o.num_bounce_blocks, t.lb, t.le, t.plan, o, out);
  }
  if (t.plan.first == KVBM_STRATEGY_MEMCPY) {
    for (int d = 0; d < nd; ++d) {
      if ((rc = host_memcpy_transfer(*t.S, *t.D[d], src_ids[d], dst_ids[d], n, o.has_layer_range != 0, t.lb, t.le))) return rc;
      m->bytes_moved += n * (t.le - t.lb) * t.S->cfg.outer_dim * t.D[d]->region;
    }
    return KVBM_OK;  // synchronous: TransferCompleteNotification::completed() (memcpy.rs:91-92)
  }
  DeviceGuard g(m->device);
  const cudaStream_t stream = pick_stream(m, t.plan.first, o);
  uint64_t seq;
  Slot* sl;
  rc = t.permute ? launch_permute(m, &t, 1, 1, src_ids, dst_ids[0], n, o, stream, &seq)
                 : launch_cuda(m, t.S, t.D, nd, src_ids, dst_ids, n, replicate, t.lb, t.le, o, stream, nullptr, &sl, &seq);
  if (rc) return rc;
  // caller-provided stream: caller manages sync, completed() is returned (cuda.rs:139-141)
  if (out) *out = o.use_caller_stream ? 0 : seq;
  return KVBM_OK;
}

// The windows of a gather, before any layout is looked up: at least one source and one window, none in the options, at most
// KVBM_GATHER_MAX_SOURCES, each naming a source, with heads, on destination heads no other window writes.  layers: a staged
// gather's windows (windows[j] is layers[j]'s head window), each with layers, whose layer windows are equal (one stage) or
// disjoint in the destination; only the windows of one stage may not share a destination head.  shared_heads: a routed gather,
// whose windows of one stage may share destination heads (its routing checks reject a sequence routed to two of them).
static int check_gather_windows(size_t num_srcs, const kvbm_layout_handle* srcs, const kvbm_head_window* windows, size_t nw,
                                const kvbm_transfer_options& o, const kvbm_shard_window* layers = nullptr, bool shared_heads = false)
{
  if (num_srcs == 0 || !srcs || !windows || nw == 0) return fail(KVBM_ERR, "a gather needs at least one source and one window");
  if (o.head_count) return fail(KVBM_ERR, "a gather takes its head windows from the windows argument: options.head_count must be 0");
  if (nw > KVBM_GATHER_MAX_SOURCES)
    return fail(KVBM_ERR_UNSUPPORTED, "a gather takes at most " + std::to_string(KVBM_GATHER_MAX_SOURCES) + " windows, got " + std::to_string(nw));
  for (size_t j = 0; j < nw; ++j) {
    if (windows[j].src_rank >= num_srcs)
      return fail(KVBM_ERR_RANGE, "window " + std::to_string(j) + " names source " + std::to_string(windows[j].src_rank) + " of " +
                                      std::to_string(num_srcs));
    if (windows[j].head_count == 0) return fail(KVBM_ERR_RANGE, "window " + std::to_string(j) + " has no heads");
    if (layers && layers[j].layer_count == 0) return fail(KVBM_ERR_RANGE, "window " + std::to_string(j) + " has no layers");
    for (size_t t = 0; t < j; ++t) {
      if (layers) {
        const kvbm_shard_window &a = layers[t], &b = layers[j];
        if (a.dst_layer_begin != b.dst_layer_begin || a.layer_count != b.layer_count) {
          if (b.dst_layer_begin < a.dst_layer_begin + a.layer_count && a.dst_layer_begin < b.dst_layer_begin + b.layer_count)
            return fail(KVBM_ERR_OVERLAP, "windows " + std::to_string(t) + " and " + std::to_string(j) +
                                              " have layer windows that partly overlap in the destination");
          continue;  // different stages may share destination heads
        }
      }
      if (shared_heads) continue;
      if (windows[j].dst_head_begin < windows[t].dst_head_begin + windows[t].head_count &&
          windows[t].dst_head_begin < windows[j].dst_head_begin + windows[j].head_count)
        return fail(KVBM_ERR_OVERLAP, "windows " + std::to_string(t) + " and " + std::to_string(j) + " overlap in the destination");
    }
  }
  return KVBM_OK;
}

// Layer window j (a kvbm_shard_window or kvbm_scatter_window) inside the source's snl layers and the destination's dnl.
template <class Window>
static int check_window_layers(const Window& w, size_t j, size_t snl, size_t dnl)
{
  if (w.src_layer_begin > snl || w.layer_count > snl - w.src_layer_begin)
    return fail(KVBM_ERR_RANGE, "window " + std::to_string(j) + "'s source layers " + std::to_string(w.src_layer_begin) + ".." +
                                    std::to_string(w.src_layer_begin + w.layer_count) + " exceed the source's num_layers " + std::to_string(snl));
  if (w.dst_layer_begin > dnl || w.layer_count > dnl - w.dst_layer_begin)
    return fail(KVBM_ERR_RANGE, "window " + std::to_string(j) + "'s destination layers " + std::to_string(w.dst_layer_begin) + ".." +
                                    std::to_string(w.dst_layer_begin + w.layer_count) + " exceed the destination's num_layers " +
                                    std::to_string(dnl));
  return KVBM_OK;
}

// Every layer of the options' range over `side`'s nl layers (the side `begin` counts) in some window; a range past them is
// rejected by the range's own check.
template <class Window>
static int check_layers_covered(const Window* w, size_t nw, size_t Window::*begin, size_t nl, const kvbm_transfer_options& o, const char* side)
{
  const size_t lb = o.has_layer_range ? o.layer_begin : 0, le = o.has_layer_range ? std::min(o.layer_end, nl) : nl;
  for (size_t l = lb; l < le; ++l) {
    bool in = false;
    for (size_t j = 0; j < nw && !in; ++j) in = l >= w[j].*begin && l - w[j].*begin < w[j].layer_count;
    if (!in) return fail(KVBM_ERR_RANGE, std::string(side) + " layer " + std::to_string(l) + " of the layer range is in no window's layers");
  }
  return KVBM_OK;
}

// What a staged gather checks of its layer windows once the windows passed check_gather_windows, under the manager's lock:
// the destination's handle, each layer window inside its source's and the destination's layers, and every destination layer of
// the options' range inside some window (KVBM_ERR_RANGE).
static int check_stage_layers(kvbm_transfer_manager* m, const kvbm_layout_handle* srcs, kvbm_layout_handle dst_h, const kvbm_shard_window* sw,
                              size_t nw, const kvbm_transfer_options& o)
{
  const Layout* D = m->find(dst_h);
  if (!D) return fail(KVBM_ERR_HANDLE, "invalid destination handle");
  const size_t dnl = D->cfg.num_layers;
  for (size_t j = 0; j < nw; ++j) {
    const Layout* S = m->find(srcs[sw[j].src_rank]);
    if (!S) return fail(KVBM_ERR_HANDLE, "invalid source handle");
    if (int rc = check_window_layers(sw[j], j, S->cfg.num_layers, dnl)) return rc;
  }
  return check_layers_covered(sw, nw, &kvbm_shard_window::dst_layer_begin, dnl, o, "destination");
}

// A TP re-shard's assembly as one hand-off: every window is validated as the windowed execute_transfer of its (source,
// destination) pair, then one permuting launch moves all of them and one signal launch writes the done flag and the
// completion word after the last byte landed.
// ls: the streamed gather, checked as above and then for its flags, launched gated on them.
// layers: a PP x TP re-shard's assembly (the staged gather), windows[j] being the head window of layers[j].  The windows are
// checked with head overlaps only within a stage and partly overlapping layer windows rejected; then check_stage_layers; then
// each pair as above but for the equal layer counts, the options' layer range being the destination's.
static int execute_gather(kvbm_transfer_manager* m, size_t num_srcs, const kvbm_layout_handle* srcs, const size_t* const* src_ids,
                          kvbm_layout_handle dst_h, const size_t* dst_ids, size_t n, const kvbm_head_window* windows, size_t nw,
                          const kvbm_transfer_options* opts_in, kvbm_notification* out, const kvbm_layer_stream* ls = nullptr,
                          const kvbm_shard_window* layers = nullptr)
{
  kvbm_transfer_options o{};
  if (opts_in) o = *opts_in;
  if (out) *out = 0;
  if (int rc = check_gather_windows(num_srcs, srcs, windows, nw, o, layers)) return rc;
  if (n && (!src_ids || !dst_ids)) return fail(KVBM_ERR, "null block id list");
  std::lock_guard<std::mutex> lk(m->mu);
  if (layers)
    if (int rc = check_stage_layers(m, srcs, dst_h, layers, nw, o)) return rc;
  Transfer e[KVBM_GATHER_MAX_SOURCES];
  for (size_t j = 0; j < nw; ++j) {
    const size_t* s = src_ids ? src_ids[windows[j].src_rank] : nullptr;
    int rc = resolve(m, srcs[windows[j].src_rank], 1, &dst_h, &s, &dst_ids, n, o, &windows[j], &e[j], layers != nullptr);
    if (rc) return rc;
    if (e[j].plan.first != e[0].plan.first) return fail(KVBM_ERR_UNSUPPORTED, "the sources of a gather need the same CUDA strategy");
  }
  if (e[0].empty) return KVBM_OK;  // nothing to move (no blocks or an empty layer range), as execute()
  if (ls)
    if (int rc = check_layer_stream_flags(m, *ls, e, nw)) return rc;

  DeviceGuard g(m->device);
  return launch_permute(m, e, nw, num_srcs, src_ids, dst_ids, n, o, pick_stream(m, e[0].plan.first, o), nullptr, out, ls, layers);
}

// Blocks a token range [tb, te) touches on a side with pages of `page` tokens: table[tb / page .. ceil(te / page)).
static size_t repage_blocks(size_t tb, size_t te, size_t page) { return tb == te ? 0 : (te + page - 1) / page - tb / page; }

// The checks of one re-paging (source, destination) pair, in this order: both layouts addressable and not both remote,
// the options re-paging takes, named formats (the options override a layout's own; filled into *src_kv / *dst_kv), head counts
// known and dividing inner_dim, check_compat's head row and cast dtypes, equal num_heads (unless `windows`: a gather's head
// windows pick the heads, so the counts may differ) and dtypes, pages that divide and the walk's rules.  staged: a staged
// re-paging gather's pair, whose layer counts may differ (check_compat's staged).  anypage: kvbm_manager_execute_repage_anypage's
// pair, whose pages need not divide but must keep the page split exact (KVBM_ERR_UNSUPPORTED).
static int check_repage_pair(const Layout& S, const Layout& D, const kvbm_transfer_options& o, bool windows, int* src_kv, int* dst_kv,
                             bool staged = false, bool anypage = false)
{
  if (S.unmapped || D.unmapped)
    return fail(KVBM_ERR_UNSUPPORTED, "a re-paging transfer needs both layouts addressable from this process (one is a descriptor of another process's host memory)");
  if (S.remote && D.remote) return fail(KVBM_ERR_UNSUPPORTED, "Both src and dst are remote - this is not supported.");
  if (o.head_count || o.layer_ready_flags || o.layer_done_flags || o.per_dst_done_flags || o.per_dst_layer_done_flags || o.multicast ||
      o.bounce_layout || o.bounce_block_ids || o.num_bounce_blocks)
    return fail(KVBM_ERR_UNSUPPORTED, "a re-paging transfer takes no head window, layer streaming, per-destination flags, multicast or bounce buffer");
  const int skv = *src_kv = o.src_kv_layout ? o.src_kv_layout : S.kv_block_layout;
  const int dkv = *dst_kv = o.dst_kv_layout ? o.dst_kv_layout : D.kv_block_layout;
  if (skv < KVBM_KV_UNIVERSAL_TP || skv > KVBM_KV_OPERATIONAL_NHD || dkv < KVBM_KV_UNIVERSAL_TP || dkv > KVBM_KV_OPERATIONAL_NHD)
    return fail(KVBM_ERR_UNSUPPORTED, std::string("re-paging needs named KV block layouts on both sides (the format decides where a token lives): src=") +
                                          kv_name(skv) + ", dst=" + kv_name(dkv));
  int rc;
  if ((rc = need_num_heads(S.cfg)) || (rc = need_num_heads(D.cfg)) || (rc = need_divisible_heads(S.cfg)) || (rc = need_divisible_heads(D.cfg)))
    return rc;
  if ((rc = check_compat(S, D, o.cast_mode, true, staged))) return rc;
  const size_t ps = S.cfg.page_size, pd = D.cfg.page_size;
  if ((!windows && S.cfg.num_heads != D.cfg.num_heads) || (o.cast_mode == KVBM_CAST_NONE && S.cfg.dtype_width_bytes != D.cfg.dtype_width_bytes))
    return fail(KVBM_ERR_INCOMPATIBLE, "a re-paging transfer needs equal num_heads, head_dim and dtype on both sides");
  if (anypage) {
    // include/kvbm_kernels.h's exactness bound, (big + small - gcd) * small < 2^32, as the unit helper applies it to an empty batch
    size_t nu, ns, nd;
    if (ps > UINT32_MAX || pd > UINT32_MAX ||
        kvbm_kernels_repage_anypage_units(nullptr, 0, static_cast<uint32_t>(ps), static_cast<uint32_t>(pd), nullptr, 0, &nu, &ns, &nd))
      return fail(KVBM_ERR_UNSUPPORTED, "page sizes src=" + std::to_string(ps) + ", dst=" + std::to_string(pd) +
                                            " are past the re-paging walk's exactness bound (big + small - gcd) * small < 2^32");
  } else if (ps % pd && pd % ps) {
    return fail(KVBM_ERR_INCOMPATIBLE, "re-paging needs one page size to divide the other: src=" + std::to_string(ps) + ", dst=" + std::to_string(pd));
  }
  return check_walk(S, D, skv, dkv, o.cast_mode);
}

// The id counts a token range implies on either side of a re-paging request.
static int check_repage_counts(size_t tb, size_t te, size_t ps, size_t pd, size_t n_src, size_t n_dst)
{
  const size_t want_src = repage_blocks(tb, te, ps), want_dst = repage_blocks(tb, te, pd);
  if (n_src != want_src || n_dst != want_dst)
    return fail(KVBM_ERR_LENGTH_MISMATCH, "tokens " + std::to_string(tb) + ".." + std::to_string(te) + " span " + std::to_string(want_src) +
                                              " source and " + std::to_string(want_dst) + " destination blocks, got src=" + std::to_string(n_src) +
                                              ", dst=" + std::to_string(n_dst));
  return KVBM_OK;
}

// The strategy of a re-paging pair: a direct CUDA one, as select_direct_strategy and resolve()'s peer rule give it.
static int repage_strategy(kvbm_transfer_manager* m, const Layout& S, const Layout& D, kvbm_transfer_plan* p)
{
  *p = kvbm_transfer_plan{};
  if (int rc = select_direct_strategy(S.storage, D.storage, &m->caps, p)) return rc;
  const bool two_hop = p->two_hop || (p->first == KVBM_STRATEGY_CUDA_ASYNC_D2D && !m->caps.allow_gpu_rdma &&
                                      (S.device_id != D.device_id || S.remote != D.remote));
  if (two_hop || !cuda_strategy(p->first))
    return fail(KVBM_ERR_UNSUPPORTED, "re-paging runs on a direct CUDA strategy only (not Memcpy, two-hop or NIXL plans)");
  return KVBM_OK;
}

// A re-paging request's checks after its pairs', in order: the token range, the layer range over `c`'s layers (*lb / *le), the
// id counts the range implies and non-null id lists.  The per-window lists follow, the caller's own.
static int check_repage_range(size_t tb, size_t te, const kvbm_layout_config& c, const kvbm_transfer_options& o, size_t ps, size_t pd, size_t n_src,
                              const void* src_ids, size_t n_dst, const void* dst_ids, size_t* lb, size_t* le)
{
  if (tb > te || te > (size_t{1} << 31))
    return fail(KVBM_ERR_RANGE, "Token range " + std::to_string(tb) + ".." + std::to_string(te) + " is reversed or reaches past 2^31 tokens");
  int rc;
  if ((rc = check_layer_range(c, o, lb, le)) || (rc = check_repage_counts(tb, te, ps, pd, n_src, n_dst))) return rc;
  if ((n_src && !src_ids) || (n_dst && !dst_ids)) return fail(KVBM_ERR, "null block id list");
  return KVBM_OK;
}

// The last checks of a request with something to move, in order: each window's direct CUDA strategy (e[j].S to e[j].D[0]) and
// one for all of them (else `mixed`, the error text), a CUDA device, the cast scales and, with ls, the flags of e[0 .. n_flagged).
static int check_repage_launch(kvbm_transfer_manager* m, Transfer* e, size_t nw, const kvbm_transfer_options& o, const kvbm_layer_stream* ls,
                               size_t n_flagged, const char* mixed)
{
  int rc;
  for (size_t j = 0; j < nw; ++j) {
    if ((rc = repage_strategy(m, *e[j].S, *e[j].D[0], &e[j].plan))) return rc;
    if (e[j].plan.first != e[0].plan.first) return fail(KVBM_ERR_UNSUPPORTED, mixed);
  }
  if ((rc = need_cuda_device(m))) return rc;
  if (o.cast_scales && (rc = check_cast_scales(m, o.cast_scales))) return rc;
  if (ls && (rc = check_layer_stream_flags(m, *ls, e, n_flagged))) return rc;
  return KVBM_OK;
}

// Re-paging hand-off: tokens [tb, te) of one sequence from the sources' block tables to the destination's, each side with its
// own page size, as one launch with one notification.  Validated on its own (resolve() assumes one page size and equal id
// counts), in the order below; a request that fails several checks reports the first.
// gather: a TP re-shard's assembly across engines with different page sizes (kvbm_manager_execute_repage_gather and its
// streamed form), execute_gather's windows over the token range.  The windows are checked as execute_gather checks them and
// the destination's handle is looked up first; every window's source is then checked against the destination as a pair
// whose head counts may differ, with its head window and with one page size for every source.  Launched as one stage over the
// destination's layers through kvbm_kernels_paged_stage_repage_gather, or its streamed form with ls.
// layers: a staged re-paging gather, a PP x TP re-shard's assembly across engines with different page sizes
// (kvbm_manager_execute_stage_repage_gather), windows[j] being the head window of layers[j].  The windows are checked as
// execute_gather checks a staged gather's, then check_stage_layers, then each pair as above but for the equal layer counts;
// the options' layer range and the cast scales are the destination's.  Launched through the same entries with its layer
// windows; each window's bytes count over its layers inside the layer range.
// Otherwise the plain re-page (kvbm_manager_execute_repage): source 0 over every head of both sides, `windows` unused.  Its
// source's handle is looked up first, its options fail the pair's checks, its head counts must be equal, and it is launched
// through kvbm_kernels_paged_repage, which has no head limit.
// A re-paging request as check_repage_request validated it: every window's Transfer, the destination, the layer range and
// whether there is nothing to move.
struct RepageRequest {
  Transfer e[KVBM_GATHER_MAX_SOURCES];
  Layout* D = nullptr;
  size_t lb = 0, le = 0;
  bool empty = false;
};

// Whether a routed gather's sequence with source mask *mask reads source r; every source without a mask.
static bool reads_source(const uint32_t* mask, size_t r) { return !mask || (r < 32 && ((*mask >> r) & 1u)); }

// Every check of a re-paging request after check_gather_windows, under the manager's lock, in the order above.  mask: a routed
// sequence's sources, whose id lists alone are read and checked.  anypage: check_repage_pair's.
static int check_repage_request(kvbm_transfer_manager* m, size_t num_srcs, const kvbm_layout_handle* srcs, const size_t* const* src_ids,
                                size_t n_src, kvbm_layout_handle dst_h, const size_t* dst_ids, size_t n_dst, size_t tb, size_t te,
                                const kvbm_head_window* windows, size_t nw, const kvbm_transfer_options& o, const kvbm_layer_stream* ls,
                                bool gather, const kvbm_shard_window* layers, RepageRequest* R, const uint32_t* mask = nullptr,
                                bool anypage = false)
{
  int rc;
  if (layers && (rc = check_stage_layers(m, srcs, dst_h, layers, nw, o))) return rc;
  Layout*& D = R->D = nullptr;
  Transfer* e = R->e;
  auto find_dst = [&] { return (D = m->find(dst_h)) ? KVBM_OK : fail(KVBM_ERR_HANDLE, "invalid destination handle"); };
  if (gather && (rc = find_dst())) return rc;  // the plain re-page looks its destination up after its source, in the loop
  for (size_t j = 0; j < nw; ++j) {
    Layout* S = e[j].S = m->find(srcs[gather ? windows[j].src_rank : 0]);
    if (!S) return fail(KVBM_ERR_HANDLE, "invalid source handle");
    if (!D && (rc = find_dst())) return rc;
    const kvbm_head_window& w = e[j].window = gather ? windows[j] : kvbm_head_window{0, 0, 0, S->cfg.num_heads};
    e[j].D[0] = D;
    if ((rc = check_repage_pair(*S, *D, o, gather, &e[j].src_kv, &e[j].dst_kv, layers != nullptr, anypage)) ||
        (rc = check_head_window(*S, *D, w, 1)))
      return rc;
    if (S->cfg.page_size != e[0].S->cfg.page_size)
      return fail(KVBM_ERR_INCOMPATIBLE, "the sources of a re-paging gather need one page size: source " + std::to_string(e[0].window.src_rank) +
                                             " has " + std::to_string(e[0].S->cfg.page_size) + ", source " + std::to_string(w.src_rank) +
                                             " has " + std::to_string(S->cfg.page_size));
  }
  const Layout& S0 = *e[0].S;
  if ((rc = check_repage_range(tb, te, layers ? D->cfg : S0.cfg, o, S0.cfg.page_size, D->cfg.page_size, n_src, src_ids, n_dst, dst_ids, &R->lb,
                               &R->le)))
    return rc;
  for (size_t j = 0; j < nw; ++j) {
    const size_t r = e[j].window.src_rank;
    if (!reads_source(mask, r)) continue;
    const size_t* s = n_src ? src_ids[r] : nullptr;
    if (n_src && !s) return fail(KVBM_ERR, "null block id list");
    if ((rc = check_block_ids(s, n_src, dst_ids, n_dst, e[j].S->cfg.num_blocks, D->cfg.num_blocks, srcs[r] == dst_h))) return rc;
  }
  if ((R->empty = tb == te || R->lb == R->le)) return KVBM_OK;  // nothing to move, as execute()
  return check_repage_launch(m, e, nw, o, ls, nw, "the sources of a gather need the same CUDA strategy");
}

// What a re-paging batch stages in its one copy: its non-empty sequences' ranges and each id list's tables, concatenated in batch
// order, and the unit table.  lists[k]: list k's table, null for a list no window uses.
struct BatchTables {
  std::vector<kvbm_repage_seq> ranges;
  std::vector<kvbm_repage_unit> units;
  std::vector<std::vector<size_t>> cat;
  std::vector<const size_t*> lists;
};

// What a re-paging request's units are, as the kernel library's re-paging launches take them: the single entries' one token
// range, or a batch of sequences whose unit table's fourth word is each unit's sequence index (kSeqs), its sequence's window mask
// (kRouted), its phase where pages need not divide (kPhased), or both (kRoutedPhased).  Each batch kind has its own unit table
// helper and kernel entries.
enum RepageUnits { kRange, kSeqs, kRouted, kPhased, kRoutedPhased };
static bool phased_units(RepageUnits k) { return k == kPhased || k == kRoutedPhased; }

// List k of sequence q is ids(q, k): q.n_src ids for k < num_src_lists, else q.n_dst.  check(t->cat), the caller's duplicate-id
// checks, runs before the unit table, which the helper of `units` writes (the same 16 B records for every kind).  routes (a
// routed kind): each non-empty sequence's range and window mask, in t->ranges' order.  *n_src / *n_dst: each concatenated source
// and destination table's length.
template <class Seq, class Ids, class Check>
static int batch_tables(const Seq* seqs, size_t num_seqs, const std::vector<bool>& used, size_t num_src_lists, uint32_t ps, uint32_t pd,
                        Ids ids, Check check, BatchTables* t, size_t* n_src, size_t* n_dst, RepageUnits units,
                        const kvbm_route_seq* routes)
{
  t->cat.resize(used.size());
  for (size_t i = 0; i < num_seqs; ++i) {
    const Seq& q = seqs[i];
    if (q.token_begin == q.token_end) continue;
    t->ranges.push_back(kvbm_repage_seq{static_cast<uint32_t>(q.token_begin), static_cast<uint32_t>(q.token_end)});
    for (size_t k = 0; k < used.size(); ++k)
      if (used[k]) t->cat[k].insert(t->cat[k].end(), ids(q, k), ids(q, k) + (k < num_src_lists ? q.n_src : q.n_dst));
  }
  if (int rc = check(t->cat)) return rc;
  static_assert(sizeof(kvbm_route_unit) == sizeof(kvbm_repage_unit) && sizeof(kvbm_repage_anypage_unit) == sizeof(kvbm_repage_unit) &&
                    sizeof(kvbm_route_anypage_unit) == sizeof(kvbm_repage_unit),
                "one staged record layout");
  auto write = [&](kvbm_repage_unit* out, size_t cap, size_t* num_units) {
    const size_t n = t->ranges.size();
    switch (units) {
      case kRouted:
        return kvbm_kernels_repage_route_units(routes, n, ps, pd, reinterpret_cast<kvbm_route_unit*>(out), cap, num_units, n_src, n_dst);
      case kPhased:
        return kvbm_kernels_repage_anypage_units(t->ranges.data(), n, ps, pd, reinterpret_cast<kvbm_repage_anypage_unit*>(out), cap, num_units,
                                                 n_src, n_dst);
      case kRoutedPhased:
        return kvbm_kernels_repage_route_anypage_units(routes, n, ps, pd, reinterpret_cast<kvbm_route_anypage_unit*>(out), cap, num_units,
                                                       n_src, n_dst);
      default:
        return kvbm_kernels_repage_batch_units(t->ranges.data(), n, ps, pd, out, cap, num_units, n_src, n_dst);
    }
  };
  size_t num_units = 0;
  if (write(nullptr, 0, &num_units)) return fail(KVBM_ERR, "the batch's token ranges and page sizes have no unit table");
  t->units.resize(num_units);
  write(t->units.data(), t->units.size(), &num_units);
  for (size_t k = 0; k < used.size(); ++k) t->lists.push_back(used[k] ? t->cat[k].data() : nullptr);
  return KVBM_OK;
}

// A re-paging request over a list of sequences, each the token range and tables of one check_repage_request: the single entries
// pass their one range as one sequence, kvbm_manager_execute_repage_batch its list (`batch`).  Every sequence is checked in
// turn and the first rejected one returns its code and text; an empty one moves nothing.  Then a batch's concatenated tables
// are checked for a destination block named twice, and one slot takes every table (and a batch's unit table) in one copy, and
// one launch moves every sequence: through the batch kind's kernel entries for a batch (units other than kRange), else the
// single range's.
// masks: a routed batch (kvbm_manager_execute_repage_batch_routed), sequence i read from the sources of masks[i] only: the
// windows of a stage may share destination heads, the routing checks run after the null sequence list, each sequence's routed id
// lists alone are checked, the destination's ids are checked against the ids of the sequences routed to a source in its
// layout, unrouted positions of the staged tables are padded with block 0, and the unit table carries each sequence's window
// mask for the routed kernel entries (kRouted, or kRoutedPhased with pages that need not divide).
// A phased kind (kvbm_manager_execute_repage_anypage, kvbm_manager_execute_repage_batch_routed_anypage): check_repage_pair's
// anypage rule.
static int execute_repage(kvbm_transfer_manager* m, size_t num_srcs, const kvbm_layout_handle* srcs, kvbm_layout_handle dst_h,
                          const kvbm_repage_batch_seq* seqs, size_t num_seqs, const kvbm_head_window* windows, size_t nw,
                          const kvbm_transfer_options* opts_in, kvbm_notification* out, const kvbm_layer_stream* ls = nullptr,
                          bool gather = true, const kvbm_shard_window* layers = nullptr, RepageUnits units = kRange,
                          const uint32_t* masks = nullptr)
{
  const bool batch = units != kRange;
  kvbm_transfer_options o{};
  if (opts_in) o = *opts_in;
  if (out) *out = 0;
  int rc;
  if (gather && (rc = check_gather_windows(num_srcs, srcs, windows, nw, o, layers, masks != nullptr))) return rc;
  if (batch && num_seqs && !seqs) return fail(KVBM_ERR, "null sequence list");
  // a routed sequence's windows: bit j for each window whose source it reads
  auto window_mask = [&](size_t i) {
    uint32_t w = 0;
    for (size_t j = 0; j < nw; ++j) w |= static_cast<uint32_t>(reads_source(masks + i, windows[j].src_rank)) << j;
    return w;
  };
  if (masks && num_srcs > 32)
    return fail(KVBM_ERR_UNSUPPORTED, "a routed gather takes at most 32 sources, got " + std::to_string(num_srcs));
  std::lock_guard<std::mutex> lk(m->mu);
  if (masks) {
    uint32_t read = 0;
    for (size_t j = 0; j < nw; ++j) read |= 1u << windows[j].src_rank;
    const Layout* Dl = m->find(dst_h);  // an invalid handle is the request checks' to report
    for (size_t i = 0; i < num_seqs; ++i) {
      const std::string at = "sequence " + std::to_string(i);
      if (masks[i] == 0) return fail(KVBM_ERR_RANGE, at + " is routed to no source");
      if (num_srcs < 32 && (masks[i] >> num_srcs) != 0)
        return fail(KVBM_ERR_RANGE, at + " is routed past the " + std::to_string(num_srcs) + " sources");
      if (masks[i] & ~read) return fail(KVBM_ERR_RANGE, at + " is routed to a source no window reads");
      const uint32_t wm = window_mask(i);
      std::vector<kvbm_shard_window> routed;
      for (size_t j = 0; j < nw; ++j) {
        if (!((wm >> j) & 1u)) continue;
        for (size_t t = 0; t < j; ++t) {
          const kvbm_shard_window &a = layers[t], &b = layers[j];
          if (((wm >> t) & 1u) && a.dst_layer_begin == b.dst_layer_begin && a.layer_count == b.layer_count &&
              b.dst_head_begin < a.dst_head_begin + a.head_count && a.dst_head_begin < b.dst_head_begin + b.head_count)
            return fail(KVBM_ERR_OVERLAP, "windows " + std::to_string(t) + " and " + std::to_string(j) + " overlap in the destination");
        }
        routed.push_back(layers[j]);
      }
      if (Dl && (rc = check_layers_covered(routed.data(), routed.size(), &kvbm_shard_window::dst_layer_begin, Dl->cfg.num_layers, o,
                                           "destination")))
        return rc;
    }
  }
  // every sequence resolves the same windows, destination and layer range: only `empty` (and the strategy, set for a
  // sequence that is not empty) is the last sequence's own
  RepageRequest R;
  bool any = false;
  uint64_t bytes = 0;
  for (size_t i = 0; i < num_seqs; ++i) {
    const kvbm_repage_batch_seq& q = seqs[i];
    const uint32_t* mask = masks ? masks + i : nullptr;
    if ((rc = check_repage_request(m, num_srcs, srcs, q.src_ids, q.n_src, dst_h, q.dst_ids, q.n_dst, q.token_begin, q.token_end, windows, nw, o,
                                   ls, gather, layers, &R, mask, phased_units(units))))
      return rc;
    if (R.empty) continue;
    any = true;
    const Layout& D = *R.D;
    const uint64_t head_bytes = D.cfg.inner_dim / D.cfg.num_heads * D.cfg.dtype_width_bytes;
    if (!mask) {
      bytes += transform_bytes(R.e, nw, layers, R.lb, R.le, q.token_end - q.token_begin, head_bytes);
      continue;
    }
    for (size_t j = 0; j < nw; ++j)  // the routed windows only
      if (reads_source(mask, windows[j].src_rank)) bytes += transform_bytes(R.e + j, 1, layers + j, R.lb, R.le, q.token_end - q.token_begin, head_bytes);
  }
  if (!any) return KVBM_OK;  // no sequences, only empty ranges or an empty layer range: nothing to move
  const Transfer* e = R.e;
  const Layout &S0 = *e[0].S, *D = R.D;
  const uint32_t ups = static_cast<uint32_t>(S0.cfg.page_size), upd = static_cast<uint32_t>(D->cfg.page_size);
  const size_t* const* src_ids = seqs[0].src_ids;
  const size_t* dst_ids = seqs[0].dst_ids;
  size_t n_src = seqs[0].n_src, n_dst = seqs[0].n_dst;
  BatchTables bt;
  std::vector<kvbm_route_seq> routes;
  if (batch) {
    std::vector<bool> used(num_srcs + 1, false);  // the sources some window reads (the others' tables may be null), the destination
    for (size_t j = 0; j < nw; ++j) used[windows[j].src_rank] = true;
    used[num_srcs] = true;
    std::vector<size_t> pad;  // a routed batch's unrouted positions: block 0, never read
    for (size_t i = 0; masks && i < num_seqs; ++i) pad.resize(std::max(pad.size(), seqs[i].n_src), 0);
    auto ids = [&](const kvbm_repage_batch_seq& q, size_t k) {
      return k == num_srcs ? q.dst_ids : reads_source(masks ? masks + (&q - seqs) : nullptr, k) ? q.src_ids[k] : pad.data();
    };
    auto unique = [&](const std::vector<std::vector<size_t>>& cat) -> int {
      const std::vector<size_t>& cd = cat[num_srcs];
      std::vector<size_t> routed;
      for (size_t j = 0; j < nw; ++j) {  // the destination's uniqueness once; a source in the destination's layout also against it
        const size_t r = windows[j].src_rank;
        const bool same = srcs[r] == dst_h;
        if (!(j == 0 || same)) continue;
        const std::vector<size_t>* cs = &cat[r];
        if (masks) {  // the ids of the sequences routed to r only
          routed.clear();
          for (size_t i = 0; i < num_seqs; ++i)
            if (seqs[i].token_begin != seqs[i].token_end && reads_source(masks + i, r))
              routed.insert(routed.end(), seqs[i].src_ids[r], seqs[i].src_ids[r] + seqs[i].n_src);
          cs = &routed;
        }
        if (int rc = check_block_ids(cs->data(), cs->size(), cd.data(), cd.size(), e[j].S->cfg.num_blocks, D->cfg.num_blocks, same))
          return rc;
      }
      return KVBM_OK;
    };
    // each non-empty sequence's range with its window mask, which the routed unit table carries
    for (size_t i = 0; masks && i < num_seqs; ++i)
      if (seqs[i].token_begin != seqs[i].token_end)
        routes.push_back(kvbm_route_seq{static_cast<uint32_t>(seqs[i].token_begin), static_cast<uint32_t>(seqs[i].token_end), window_mask(i)});
    if ((rc = batch_tables(seqs, num_seqs, used, num_srcs, ups, upd, ids, unique, &bt, &n_src, &n_dst, units, routes.data())))
      return rc;
    src_ids = bt.lists.data();
    dst_ids = bt.lists[num_srcs];
  }

  DeviceGuard g(m->device);
  const cudaStream_t stream = pick_stream(m, e[0].plan.first, o);
  const uint32_t row = static_cast<uint32_t>(S0.cfg.inner_dim / S0.cfg.num_heads * S0.cfg.dtype_width_bytes);
  const uint32_t dnh = static_cast<uint32_t>(D->cfg.num_heads);
  const uint32_t utb = static_cast<uint32_t>(seqs[0].token_begin), ute = static_cast<uint32_t>(seqs[0].token_end);
  const int ilb = static_cast<int>(R.lb), ile = static_cast<int>(R.le), k = static_cast<int>(nw);
  auto launch = [&](const kvbm_permute_source* ks, const kvbm_permute_side& kd, const kvbm_permute_stream* st, const Slot& sl, uint64_t seq) {
    const uint32_t value = static_cast<uint32_t>(seq);
    if (!gather)
      return checked(kvbm_kernels_paged_repage(&ks[0].side, ups, &kd, upd, utb, ute, ilb, ile, ks[0].num_heads, row, o.cast_mode, o.cast_scales,
                                               o.done_flag, o.epoch, sl.host_flag, value, stream),
                     "kvbm_kernels_paged_repage");
    kvbm_stage_source ss[KVBM_GATHER_MAX_SOURCES] = {};
    stage_sources(ks, layers, nw, D->cfg.num_layers, ss);
    // a batch: its kind's entry, streamed or not
    const int32_t* du = sl.dev_ids + units_at(num_srcs * n_src + n_dst);
    auto run = [&](auto entry, auto streamed_entry, const char* name, const char* streamed_name, const auto* qs, size_t n, const auto* t) {
      if (st)
        return checked(streamed_entry(ss, k, ups, &kd, dnh, upd, qs, n, t, bt.units.size(), ilb, ile, row, o.cast_mode, o.cast_scales, st, stream),
                       streamed_name);
      return checked(entry(ss, k, ups, &kd, dnh, upd, qs, n, t, bt.units.size(), ilb, ile, row, o.cast_mode, o.cast_scales, o.done_flag, o.epoch,
                           sl.host_flag, value, stream),
                     name);
    };
    switch (units) {
      case kSeqs:
        return run(kvbm_kernels_paged_stage_repage_gather_batch, kvbm_kernels_paged_stage_repage_gather_batch_streamed,
                   "kvbm_kernels_paged_stage_repage_gather_batch", "kvbm_kernels_paged_stage_repage_gather_batch_streamed", bt.ranges.data(),
                   bt.ranges.size(), reinterpret_cast<const kvbm_repage_unit*>(du));
      case kRouted:
        return run(kvbm_kernels_paged_stage_repage_gather_routed, kvbm_kernels_paged_stage_repage_gather_routed_streamed,
                   "kvbm_kernels_paged_stage_repage_gather_routed", "kvbm_kernels_paged_stage_repage_gather_routed_streamed", routes.data(),
                   routes.size(), reinterpret_cast<const kvbm_route_unit*>(du));
      case kPhased:
        return run(kvbm_kernels_paged_stage_repage_gather_anypage, kvbm_kernels_paged_stage_repage_gather_anypage_streamed,
                   "kvbm_kernels_paged_stage_repage_gather_anypage", "kvbm_kernels_paged_stage_repage_gather_anypage_streamed",
                   bt.ranges.data(), bt.ranges.size(), reinterpret_cast<const kvbm_repage_anypage_unit*>(du));
      case kRoutedPhased:
        return run(kvbm_kernels_paged_stage_repage_gather_routed_anypage, kvbm_kernels_paged_stage_repage_gather_routed_anypage_streamed,
                   "kvbm_kernels_paged_stage_repage_gather_routed_anypage", "kvbm_kernels_paged_stage_repage_gather_routed_anypage_streamed",
                   routes.data(), routes.size(), reinterpret_cast<const kvbm_route_anypage_unit*>(du));
      case kRange:
        break;
    }
    if (st)
      return checked(kvbm_kernels_paged_stage_repage_gather_streamed(ss, k, ups, &kd, dnh, upd, utb, ute, ilb, ile, row, o.cast_mode,
                                                                     o.cast_scales, st, stream),
                     "kvbm_kernels_paged_stage_repage_gather_streamed");
    return checked(kvbm_kernels_paged_stage_repage_gather(ss, k, ups, &kd, dnh, upd, utb, ute, ilb, ile, row, o.cast_mode, o.cast_scales,
                                                          o.done_flag, o.epoch, sl.host_flag, value, stream),
                   "kvbm_kernels_paged_stage_repage_gather");
  };
  return launch_transform(m, e, nw, num_srcs, src_ids, n_src, dst_ids, n_dst, ls, o, stream, bytes, nullptr, out, launch, bt.units.data(),
                          bt.units.size());
}

// The windows of a scatter, before any layout is looked up: at least one destination and one window, none in the options, at most
// KVBM_GATHER_MAX_SOURCES, each naming a destination, with heads and layers; source layer windows equal (one stage) or disjoint;
// the windows of one destination on disjoint (layer, head) rectangles of it; no destination handle listed twice.
static int check_scatter_windows(size_t num_dsts, const kvbm_layout_handle* dsts, const kvbm_scatter_window* w, size_t nw,
                                 const kvbm_transfer_options& o)
{
  if (num_dsts == 0 || !dsts || !w || nw == 0) return fail(KVBM_ERR, "a scatter needs at least one destination and one window");
  if (o.head_count) return fail(KVBM_ERR, "a scatter takes its head windows from the windows argument: options.head_count must be 0");
  if (nw > KVBM_GATHER_MAX_SOURCES)
    return fail(KVBM_ERR_UNSUPPORTED, "a scatter takes at most " + std::to_string(KVBM_GATHER_MAX_SOURCES) + " windows, got " + std::to_string(nw));
  auto meet = [](size_t a, size_t na, size_t b, size_t nb) { return a < b + nb && b < a + na; };
  for (size_t j = 0; j < nw; ++j) {
    if (w[j].dst_rank >= num_dsts)
      return fail(KVBM_ERR_RANGE, "window " + std::to_string(j) + " names destination " + std::to_string(w[j].dst_rank) + " of " +
                                      std::to_string(num_dsts));
    if (w[j].head_count == 0) return fail(KVBM_ERR_RANGE, "window " + std::to_string(j) + " has no heads");
    if (w[j].layer_count == 0) return fail(KVBM_ERR_RANGE, "window " + std::to_string(j) + " has no layers");
    for (size_t t = 0; t < j; ++t) {
      const bool same = w[t].src_layer_begin == w[j].src_layer_begin && w[t].layer_count == w[j].layer_count;
      if (!same && meet(w[t].src_layer_begin, w[t].layer_count, w[j].src_layer_begin, w[j].layer_count))
        return fail(KVBM_ERR_OVERLAP, "windows " + std::to_string(t) + " and " + std::to_string(j) + " have source layer windows that partly overlap");
      if (w[t].dst_rank == w[j].dst_rank && meet(w[t].dst_layer_begin, w[t].layer_count, w[j].dst_layer_begin, w[j].layer_count) &&
          meet(w[t].dst_head_begin, w[t].head_count, w[j].dst_head_begin, w[j].head_count))
        return fail(KVBM_ERR_OVERLAP, "windows " + std::to_string(t) + " and " + std::to_string(j) + " overlap in destination " +
                                          std::to_string(w[j].dst_rank));
    }
  }
  for (size_t d = 0; d < num_dsts; ++d)
    for (size_t e = 0; e < d; ++e)
      if (dsts[d] == dsts[e]) return fail(KVBM_ERR_OVERLAP, "destinations " + std::to_string(e) + " and " + std::to_string(d) + " are one layout");
  return KVBM_OK;
}

// A scatter request as check_scatter_request validated it: the source, the destinations, every window's Transfer, the layer range
// and whether there is nothing to move.
struct ScatterRequest {
  Layout* S = nullptr;
  std::vector<Layout*> D;
  Transfer e[KVBM_GATHER_MAX_SOURCES];
  size_t lb = 0, le = 0;
  bool empty = false;
};

// Whether a routed scatter's sequence with destination mask *mask goes to destination d; every destination without a mask.
static bool routed_to(const uint32_t* mask, size_t d) { return !mask || (d < 32 && ((*mask >> d) & 1u)); }

// Every check of one sequence of a scatter after check_scatter_windows, under the manager's lock, in the order its header gives.
// mask: a routed sequence's destinations, whose id lists alone are read and checked.  anypage: check_repage_pair's.
static int check_scatter_request(kvbm_transfer_manager* m, kvbm_layout_handle src_h, const kvbm_scatter_batch_seq& q, size_t num_dsts,
                                 const kvbm_layout_handle* dsts, const kvbm_scatter_window* w, size_t nw, const kvbm_transfer_options& o,
                                 const kvbm_layer_stream* ls, ScatterRequest* R, const uint32_t* mask = nullptr, bool anypage = false)
{
  int rc;
  Layout* S = R->S = m->find(src_h);
  if (!S) return fail(KVBM_ERR_HANDLE, "invalid source handle");
  std::vector<Layout*>& D = R->D;
  D.assign(num_dsts, nullptr);
  for (size_t d = 0; d < num_dsts; ++d)
    if (!(D[d] = m->find(dsts[d]))) return fail(KVBM_ERR_HANDLE, "invalid destination handle");
  for (size_t j = 0; j < nw; ++j)
    if ((rc = check_window_layers(w[j], j, S->cfg.num_layers, D[w[j].dst_rank]->cfg.num_layers))) return rc;
  if ((rc = check_layers_covered(w, nw, &kvbm_scatter_window::src_layer_begin, S->cfg.num_layers, o, "source"))) return rc;
  // the pair checks take the per-destination done flags, which a scatter honours, as absent
  kvbm_transfer_options op = o;
  op.per_dst_done_flags = nullptr;
  Transfer* e = R->e;
  for (size_t j = 0; j < nw; ++j) {
    Layout& Dj = *D[w[j].dst_rank];
    e[j].S = S;
    e[j].D[0] = &Dj;
    e[j].window = kvbm_head_window{0, w[j].src_head_begin, w[j].dst_head_begin, w[j].head_count};
    if ((rc = check_repage_pair(*S, Dj, op, true, &e[j].src_kv, &e[j].dst_kv, true, anypage)) || (rc = check_head_window(*S, Dj, e[j].window, 1)))
      return rc;
    if (Dj.cfg.page_size != D[w[0].dst_rank]->cfg.page_size)
      return fail(KVBM_ERR_INCOMPATIBLE, "the destinations of a scatter need one page size: destination " + std::to_string(w[0].dst_rank) +
                                             " has " + std::to_string(D[w[0].dst_rank]->cfg.page_size) + ", destination " +
                                             std::to_string(w[j].dst_rank) + " has " + std::to_string(Dj.cfg.page_size));
  }
  const size_t tb = q.token_begin, te = q.token_end;
  if ((rc = check_repage_range(tb, te, S->cfg, o, S->cfg.page_size, D[w[0].dst_rank]->cfg.page_size, q.n_src, q.src_ids, q.n_dst, q.dst_ids,
                               &R->lb, &R->le)))
    return rc;
  for (size_t j = 0; j < nw; ++j) {
    const size_t d = w[j].dst_rank;
    if (!routed_to(mask, d)) continue;
    if (q.n_dst && !q.dst_ids[d]) return fail(KVBM_ERR, "null block id list");
    if ((rc = check_block_ids(q.src_ids, q.n_src, q.n_dst ? q.dst_ids[d] : nullptr, q.n_dst, S->cfg.num_blocks, D[d]->cfg.num_blocks,
                              src_h == dsts[d])))
      return rc;
  }
  if ((R->empty = tb == te || R->lb == R->le)) return KVBM_OK;  // nothing to move, as execute()
  return check_repage_launch(m, e, nw, o, ls, 1, "the destinations of a scatter need the same CUDA strategy");
}

// One prefill rank's KV into every decode rank that needs it over a list of sequences, each the token range and tables of one
// check_scatter_request: kvbm_manager_execute_repage_scatter and its streamed form pass their one range as one sequence,
// kvbm_manager_execute_repage_scatter_batch its list (`batch`).  Every sequence is checked in turn and the first rejected one
// returns its code and text; an empty one moves nothing.  Then a batch's concatenated tables are checked per destination for a
// block named twice, and one staged copy takes [source ids, destination 0 .. num_dsts - 1 ids (the same count each)] (and a
// batch's unit table), then one launch whose signal writes the per-destination done flags and the completion word, and the
// options' done flag after it.  ls: the streamed scatter (its shape checked by the caller); the slot also holds the gate's
// workspace over the source's layers, and the one streamed launch writes every flag, the options' done flag included.
// masks: a routed batch (kvbm_manager_execute_repage_scatter_routed), sequence i going to the destinations of masks[i] only: the
// routing checks run after the windows', each sequence's routed id lists alone are checked, the uniqueness per destination runs
// over its routed sequences, unrouted positions of the staged tables are padded with block 0, and the unit table carries each
// sequence's window mask for the routed kernel entries (kRouted, or kRoutedPhased with pages that need not divide).
// A phased kind (kvbm_manager_execute_repage_scatter_anypage, kvbm_manager_execute_repage_scatter_routed_anypage):
// check_repage_pair's anypage rule.  units: as execute_repage's.
static int execute_repage_scatter(kvbm_transfer_manager* m, kvbm_layout_handle src_h, size_t num_dsts, const kvbm_layout_handle* dsts,
                                  const kvbm_scatter_batch_seq* seqs, size_t num_seqs, const kvbm_scatter_window* w, size_t nw,
                                  const kvbm_transfer_options* opts_in, kvbm_notification* out, const kvbm_layer_stream* ls = nullptr,
                                  RepageUnits units = kRange, const uint32_t* masks = nullptr)
{
  const bool batch = units != kRange;
  kvbm_transfer_options o{};
  if (opts_in) o = *opts_in;
  if (out) *out = 0;
  int rc;
  if ((rc = check_scatter_windows(num_dsts, dsts, w, nw, o))) return rc;
  if (batch && num_seqs && !seqs) return fail(KVBM_ERR, "null sequence list");
  if (masks) {
    if (num_dsts > 32)
      return fail(KVBM_ERR_UNSUPPORTED, "a routed scatter takes at most 32 destinations, got " + std::to_string(num_dsts));
    uint32_t written = 0;
    for (size_t j = 0; j < nw; ++j) written |= 1u << w[j].dst_rank;
    for (size_t i = 0; i < num_seqs; ++i) {
      const std::string at = "sequence " + std::to_string(i);
      if (masks[i] == 0) return fail(KVBM_ERR_RANGE, at + " is routed to no destination");
      if (num_dsts < 32 && (masks[i] >> num_dsts) != 0)
        return fail(KVBM_ERR_RANGE, at + " is routed past the " + std::to_string(num_dsts) + " destinations");
      if (masks[i] & ~written) return fail(KVBM_ERR_RANGE, at + " is routed to a destination no window writes");
    }
  }
  std::lock_guard<std::mutex> lk(m->mu);
  // every sequence resolves the same source, destinations, windows and layer range: only `empty` is the last sequence's own
  ScatterRequest R;
  bool any = false;
  uint64_t bytes = 0;
  for (size_t i = 0; i < num_seqs; ++i) {
    const kvbm_scatter_batch_seq& q = seqs[i];
    const uint32_t* mask = masks ? masks + i : nullptr;
    if ((rc = check_scatter_request(m, src_h, q, num_dsts, dsts, w, nw, o, ls, &R, mask, phased_units(units)))) return rc;
    if (R.empty) continue;
    any = true;
    // what lands: each routed window's destination bytes over its layers inside the range
    for (size_t j = 0; j < nw; ++j) {
      if (!routed_to(mask, w[j].dst_rank)) continue;
      const Layout& Dj = *R.e[j].D[0];
      const size_t from = std::max(R.lb, w[j].src_layer_begin), to = std::min(R.le, w[j].src_layer_begin + w[j].layer_count);
      if (to > from)
        bytes += (q.token_end - q.token_begin) * (to - from) * Dj.cfg.outer_dim * w[j].head_count *
                 (Dj.cfg.inner_dim / Dj.cfg.num_heads * Dj.cfg.dtype_width_bytes);
    }
  }
  if (!any) return KVBM_OK;  // no sequences, only empty ranges or an empty layer range: nothing to move
  const Transfer* e = R.e;
  const Layout* S = R.S;
  const std::vector<Layout*>& D = R.D;
  const size_t snl = S->cfg.num_layers;
  const uint32_t ups = static_cast<uint32_t>(S->cfg.page_size), upd = static_cast<uint32_t>(D[w[0].dst_rank]->cfg.page_size);
  const size_t* src_ids = seqs[0].src_ids;
  const size_t* const* dst_ids = seqs[0].dst_ids;
  size_t n_src = seqs[0].n_src, n_dst = seqs[0].n_dst;
  BatchTables bt;
  std::vector<kvbm_route_seq> routes;
  if (batch) {
    std::vector<bool> used(1 + num_dsts, false);  // the source, the destinations some window writes (the others' tables may be null)
    used[0] = true;
    for (size_t j = 0; j < nw; ++j) used[1 + w[j].dst_rank] = true;
    std::vector<size_t> pad;  // a routed batch's unrouted positions: block 0, never read
    for (size_t i = 0; masks && i < num_seqs; ++i) pad.resize(std::max(pad.size(), seqs[i].n_dst), 0);
    auto ids = [&](const kvbm_scatter_batch_seq& q, size_t k) {
      return !k ? q.src_ids : routed_to(masks ? masks + (&q - seqs) : nullptr, k - 1) ? q.dst_ids[k - 1] : pad.data();
    };
    auto unique = [&](const std::vector<std::vector<size_t>>& cat) -> int {
      std::vector<size_t> routed;
      for (size_t d = 0; d < num_dsts; ++d) {
        if (!used[1 + d]) continue;
        const std::vector<size_t>* cd = &cat[1 + d];
        if (masks) {  // the ids of the sequences routed to d only
          routed.clear();
          for (size_t i = 0; i < num_seqs; ++i)
            if (seqs[i].token_begin != seqs[i].token_end && routed_to(masks + i, d))
              routed.insert(routed.end(), seqs[i].dst_ids[d], seqs[i].dst_ids[d] + seqs[i].n_dst);
          cd = &routed;
        }
        if (int rc = check_block_ids(cat[0].data(), cat[0].size(), cd->data(), cd->size(), S->cfg.num_blocks, D[d]->cfg.num_blocks,
                                     src_h == dsts[d]))
          return rc;
      }
      return KVBM_OK;
    };
    // each non-empty sequence's range with its window mask, which the routed unit table carries
    for (size_t i = 0; masks && i < num_seqs; ++i) {
      if (seqs[i].token_begin == seqs[i].token_end) continue;
      uint32_t targets = 0;
      for (size_t j = 0; j < nw; ++j) targets |= static_cast<uint32_t>(routed_to(masks + i, w[j].dst_rank)) << j;
      routes.push_back(kvbm_route_seq{static_cast<uint32_t>(seqs[i].token_begin), static_cast<uint32_t>(seqs[i].token_end), targets});
    }
    if ((rc = batch_tables(seqs, num_seqs, used, 1, ups, upd, ids, unique, &bt, &n_src, &n_dst, units, routes.data()))) return rc;
    src_ids = bt.lists[0];
    dst_ids = bt.lists.data() + 1;
  }

  DeviceGuard g(m->device);
  const cudaStream_t stream = pick_stream(m, e[0].plan.first, o);
  std::vector<const size_t*> lists(num_dsts + 1);
  std::vector<size_t> lens(num_dsts + 1, n_dst);
  lists[0] = src_ids;
  lens[0] = n_src;
  for (size_t d = 0; d < num_dsts; ++d) lists[1 + d] = n_dst ? dst_ids[d] : nullptr;
  Slot* sl;
  uint64_t seq;
  if ((rc = stage_ids(m, lists.data(), lens.data(), num_dsts + 1, ls ? snl + 4 : 4, stream, nullptr, &sl, &seq, bt.units.data(), bt.units.size())))
    return rc;
  const kvbm_permute_side ks{descriptor(*S), sl->dev_ids, e[0].src_kv};
  kvbm_scatter_target kt[KVBM_GATHER_MAX_SOURCES] = {};
  for (size_t j = 0; j < nw; ++j) {
    const size_t d = w[j].dst_rank;
    kt[j] = kvbm_scatter_target{{descriptor(*D[d]), sl->dev_ids + n_src + d * n_dst, e[j].dst_kv}, static_cast<uint32_t>(D[d]->cfg.num_heads),
                                static_cast<uint32_t>(w[j].src_head_begin), static_cast<uint32_t>(w[j].dst_head_begin),
                                static_cast<uint32_t>(w[j].head_count), static_cast<uint32_t>(w[j].src_layer_begin),
                                static_cast<uint32_t>(w[j].dst_layer_begin), static_cast<uint32_t>(w[j].layer_count),
                                o.per_dst_done_flags ? o.per_dst_done_flags[d] : nullptr};
  }
  const uint32_t row = static_cast<uint32_t>(S->cfg.inner_dim / S->cfg.num_heads * S->cfg.dtype_width_bytes);
  const uint32_t snh = static_cast<uint32_t>(S->cfg.num_heads);
  const uint32_t utb = static_cast<uint32_t>(seqs[0].token_begin), ute = static_cast<uint32_t>(seqs[0].token_end);
  const int k = static_cast<int>(nw), ilb = static_cast<int>(R.lb), ile = static_cast<int>(R.le);
  const int32_t* du = sl->dev_ids + units_at(n_src + num_dsts * n_dst);
  const kvbm_permute_stream st = ls ? layer_stream(*ls, e, 1, o, *sl, seq) : kvbm_permute_stream{};
  // a batch: its kind's entry, streamed or not
  auto run = [&](auto entry, auto streamed_entry, const char* name, const char* streamed_name, const auto* qs, size_t n, const auto* t) {
    if (ls)
      return checked(streamed_entry(&ks, snh, ups, kt, k, upd, qs, n, t, bt.units.size(), ilb, ile, row, o.cast_mode, o.cast_scales, &st, stream),
                     streamed_name);
    return checked(entry(&ks, snh, ups, kt, k, upd, qs, n, t, bt.units.size(), ilb, ile, row, o.cast_mode, o.cast_scales, o.epoch, sl->host_flag,
                         static_cast<uint32_t>(seq), stream),
                   name);
  };
  switch (units) {
    case kRange:
      rc = ls ? checked(kvbm_kernels_paged_repage_scatter_streamed(&ks, snh, ups, kt, k, upd, utb, ute, ilb, ile, row, o.cast_mode, o.cast_scales,
                                                                   &st, stream),
                        "kvbm_kernels_paged_repage_scatter_streamed")
              : checked(kvbm_kernels_paged_repage_scatter(&ks, snh, ups, kt, k, upd, utb, ute, ilb, ile, row, o.cast_mode, o.cast_scales, o.epoch,
                                                          sl->host_flag, static_cast<uint32_t>(seq), stream),
                        "kvbm_kernels_paged_repage_scatter");
      break;
    case kSeqs:
      rc = run(kvbm_kernels_paged_repage_scatter_batch, kvbm_kernels_paged_repage_scatter_batch_streamed, "kvbm_kernels_paged_repage_scatter_batch",
               "kvbm_kernels_paged_repage_scatter_batch_streamed", bt.ranges.data(), bt.ranges.size(), reinterpret_cast<const kvbm_repage_unit*>(du));
      break;
    case kRouted:
      rc = run(kvbm_kernels_paged_repage_scatter_routed, kvbm_kernels_paged_repage_scatter_routed_streamed, "kvbm_kernels_paged_repage_scatter_routed",
               "kvbm_kernels_paged_repage_scatter_routed_streamed", routes.data(), routes.size(), reinterpret_cast<const kvbm_route_unit*>(du));
      break;
    case kPhased:
      rc = run(kvbm_kernels_paged_repage_scatter_anypage, kvbm_kernels_paged_repage_scatter_anypage_streamed,
               "kvbm_kernels_paged_repage_scatter_anypage", "kvbm_kernels_paged_repage_scatter_anypage_streamed", bt.ranges.data(),
               bt.ranges.size(), reinterpret_cast<const kvbm_repage_anypage_unit*>(du));
      break;
    case kRoutedPhased:
      rc = run(kvbm_kernels_paged_repage_scatter_routed_anypage, kvbm_kernels_paged_repage_scatter_routed_anypage_streamed,
               "kvbm_kernels_paged_repage_scatter_routed_anypage", "kvbm_kernels_paged_repage_scatter_routed_anypage_streamed", routes.data(),
               routes.size(), reinterpret_cast<const kvbm_route_anypage_unit*>(du));
      break;
  }
  if (!rc && !ls && o.done_flag) rc = checked(kvbm_kernels_set_flags(o.done_flag, 0, 1, o.epoch, stream), "kvbm_kernels_set_flags");
  if (rc) return rc;
  if ((rc = finish_slot(m, sl, stream, bytes))) return rc;
  if (out) *out = o.use_caller_stream ? 0 : seq;
  return KVBM_OK;
}

}  // namespace kvbm_host

// =====================================================================================================
// C ABI
// =====================================================================================================
extern "C" const char* kvbm_last_error(void) { return g_last_error.c_str(); }

extern "C" int kvbm_layout_config_validate(const kvbm_layout_config* cfg)
{
  return guarded([&]() -> int {
  if (!cfg) return fail(KVBM_ERR, "null config");
  std::string why;
  int rc = validate_config(*cfg, &why);
  return rc ? fail(rc, why) : KVBM_OK;
  });
}
extern "C" size_t kvbm_layout_required_bytes(const kvbm_layout_config* cfg) { return cfg ? required_bytes(*cfg) : 0; }
extern "C" size_t kvbm_layout_bytes_per_block(const kvbm_layout_config* cfg) { return cfg ? bytes_per_block(*cfg) : 0; }

extern "C" int kvbm_select_direct_strategy(int src_kind, int dst_kind, const kvbm_transfer_capabilities* caps, kvbm_transfer_plan* out)
{
  return guarded([&]() -> int {
  if (!out) return fail(KVBM_ERR, "null plan");
  return select_direct_strategy(src_kind, dst_kind, caps, out);
  });
}

extern "C" int kvbm_select_direct_strategy_remote(int src_kind, int dst_kind, int dst_is_remote, const kvbm_transfer_capabilities* caps,
                                                  kvbm_transfer_plan* out)
{
  return guarded([&]() -> int {
  if (!out) return fail(KVBM_ERR, "null plan");
  return select_direct_strategy(src_kind, dst_kind, caps, out, dst_is_remote != 0);
  });
}

extern "C" int kvbm_select_strategy(int src_kind, int src_is_local, int dst_kind, int dst_is_local, const kvbm_transfer_capabilities* caps,
                                    kvbm_transfer_plan* out)
{
  return guarded([&]() -> int {
  if (!out) return fail(KVBM_ERR, "null plan");
  return select_strategy(src_kind, src_is_local != 0, dst_kind, dst_is_local != 0, caps, out);
  });
}

extern "C" int kvbm_manager_select_strategy(kvbm_transfer_manager* m, kvbm_layout_handle src, kvbm_layout_handle dst, kvbm_transfer_plan* out)
{
  return guarded([&]() -> int {
  if (!m || !out) return fail(KVBM_ERR, "null argument");
  std::lock_guard<std::mutex> lk(m->mu);
  Layout *S = m->find(src), *D = m->find(dst);
  if (!S || !D) return fail(KVBM_ERR_HANDLE, "invalid layout handle");
  return select_strategy(S->storage, !S->remote, D->storage, !D->remote, &m->caps, out);
  });
}

extern "C" int kvbm_validate_block_transfer(const size_t* src_ids, size_t n_src, const size_t* dst_ids, size_t n_dst,
                                            size_t src_num_blocks, size_t dst_num_blocks, int same_layout)
{
  return guarded([&]() -> int {
  return validate_block_transfer(src_ids, n_src, dst_ids, n_dst, src_num_blocks, dst_num_blocks, same_layout != 0);
  });
}

extern "C" int kvbm_manager_create(int cuda_device_id, uint64_t worker_id, kvbm_transfer_manager** out)
{
  return guarded([&]() -> int {
  if (!out) return fail(KVBM_ERR, "null out");
  auto m = std::make_unique<kvbm_transfer_manager>();
  m->device = cuda_device_id;
  m->worker_id = worker_id & 0xffffffffffffull;
  if (cuda_device_id >= 0) {
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e != cudaSuccess) return fail_cuda(e, "cudaGetDeviceCount");
    if (cuda_device_id >= count) return fail(KVBM_ERR_CUDA, "CUDA device " + std::to_string(cuda_device_id) + " does not exist");
    DeviceGuard g(cuda_device_id);
    for (int i = 0; i < kStreams; ++i) {
      CU(cudaStreamCreateWithFlags(&m->h2d[i], cudaStreamNonBlocking));
      CU(cudaStreamCreateWithFlags(&m->d2h[i], cudaStreamNonBlocking));
    }
    int rc = provision_slots(m.get());
    if (rc) return rc;
  }
  *out = m.release();
  return KVBM_OK;
  });
}

extern "C" void kvbm_manager_destroy(kvbm_transfer_manager* m)
{
  if (!m) return;
  if (m->device >= 0) {
    DeviceGuard g(m->device);
    cudaDeviceSynchronize();
    for (auto& kv : m->layouts)
      if (kv.second->dev_layer_base) cudaFree(kv.second->dev_layer_base);
    for (auto& kv : m->ipc_cache) cudaIpcCloseMemHandle(kv.second);
    for (auto& s : m->slots) {
      if (s.ev) cudaEventDestroy(s.ev);
      if (s.owns_ids && s.pinned_ids) cudaFreeHost(s.pinned_ids);
      if (s.owns_ids && s.dev_ids) cudaFree(s.dev_ids);
      if (s.owns_flag && s.host_flag) cudaFreeHost(s.host_flag);
      if (s.owns_ws && s.dev_ws) cudaFree(s.dev_ws);
    }
    if (m->pinned_arena) cudaFreeHost(m->pinned_arena);
    if (m->dev_arena) cudaFree(m->dev_arena);
    for (int i = 0; i < kStreams; ++i) {
      if (m->h2d[i]) cudaStreamDestroy(m->h2d[i]);
      if (m->d2h[i]) cudaStreamDestroy(m->d2h[i]);
    }
  }
  delete m;
}

static int finish_register(kvbm_transfer_manager* m, Layout&& L, int storage_kind, int device_id, kvbm_layout_handle* out)
{
  if (storage_kind < KVBM_STORAGE_SYSTEM || storage_kind > KVBM_STORAGE_DISK) return fail(KVBM_ERR, "unknown StorageKind");
  if (L.region >= (1ull << 32)) return fail(KVBM_ERR_CONFIG, "a (block, layer, outer) region must be < 4 GiB");
  L.storage = storage_kind;
  L.device_id = device_id;
  int rc = upload_layer_base(m, &L);
  if (rc) return rc;
  uint64_t* dev_table = L.dev_layer_base;
  *out = add_layout(m, std::move(L));
  if (*out == 0) {
    if (dev_table) cudaFree(dev_table);
    return fail(KVBM_ERR, "layout id space exhausted: 65535 layouts are registered on this worker");
  }
  return KVBM_OK;
}

extern "C" int kvbm_manager_register_fully_contiguous(kvbm_transfer_manager* m, const kvbm_layout_config* cfg, void* base, size_t size,
                                                      int storage_kind, int device_id, kvbm_layout_handle* out)
{
  return guarded([&]() -> int {
  if (!m || !cfg || !out) return fail(KVBM_ERR, "null argument");
  Layout L;
  std::string why;
  int rc = make_fully_contiguous(*cfg, reinterpret_cast<uintptr_t>(base), size, &L, &why);
  if (rc) return fail(rc, why);
  return finish_register(m, std::move(L), storage_kind, device_id, out);
  });
}

extern "C" int kvbm_manager_register_layer_separate(kvbm_transfer_manager* m, const kvbm_layout_config* cfg, void* const* layer_bases,
                                                    const size_t* layer_sizes, int block_dim, int storage_kind, int device_id,
                                                    kvbm_layout_handle* out)
{
  return guarded([&]() -> int {
  if (!m || !cfg || !out || !layer_bases || !layer_sizes) return fail(KVBM_ERR, "null argument");
  std::vector<uintptr_t> bases(cfg->num_layers);
  for (size_t i = 0; i < cfg->num_layers; ++i) bases[i] = reinterpret_cast<uintptr_t>(layer_bases[i]);
  Layout L;
  std::string why;
  int rc = make_layer_separate(*cfg, bases.data(), layer_sizes, cfg->num_layers, block_dim, &L, &why);
  if (rc) return fail(rc, why);
  return finish_register(m, std::move(L), storage_kind, device_id, out);
  });
}

extern "C" int kvbm_manager_unregister(kvbm_transfer_manager* m, kvbm_layout_handle h)
{
  return guarded([&]() -> int {
  if (!m) return fail(KVBM_ERR, "null manager");
  std::lock_guard<std::mutex> lk(m->mu);
  auto it = m->layouts.find(h);
  if (it == m->layouts.end()) return fail(KVBM_ERR_HANDLE, "invalid handle");
  if (m->device >= 0) {
    DeviceGuard g(m->device);
    for (auto& s : m->slots)
      if (s.in_flight) {
        cudaEventSynchronize(s.ev);
        s.in_flight = false;
      }
    if (it->second->dev_layer_base) cudaFree(it->second->dev_layer_base);
  }
  m->layouts.erase(it);
  return KVBM_OK;
  });
}

extern "C" int kvbm_layout_memory_region(kvbm_transfer_manager* m, kvbm_layout_handle h, size_t block, size_t layer, size_t outer,
                                         uintptr_t* addr, size_t* size)
{
  return guarded([&]() -> int {
  if (!m || !addr) return fail(KVBM_ERR, "null argument");
  std::lock_guard<std::mutex> lk(m->mu);
  Layout* L = m->find(h);
  if (!L) return fail(KVBM_ERR_HANDLE, "invalid handle");
  std::string why;
  int rc = L->memory_region(block, layer, outer, addr, size, &why);
  return rc ? fail(rc, why) : KVBM_OK;
  });
}

extern "C" int kvbm_layout_is_fully_contiguous(kvbm_transfer_manager* m, kvbm_layout_handle h)
{
  if (!m) return -1;
  std::lock_guard<std::mutex> lk(m->mu);
  Layout* L = m->find(h);
  return L ? (L->fully_contiguous ? 1 : 0) : -1;
}

extern "C" int kvbm_manager_enable_peer_access(kvbm_transfer_manager* m, int peer_device)
{
  return guarded([&]() -> int {
  if (!m || m->device < 0) return fail(KVBM_ERR_CUDA, "manager has no CUDA device");
  if (peer_device == m->device) return KVBM_OK;
  DeviceGuard g(m->device);
  int can = 0;
  CU(cudaDeviceCanAccessPeer(&can, m->device, peer_device));
  if (!can) return fail(KVBM_ERR_UNSUPPORTED, "device " + std::to_string(m->device) + " cannot map device " + std::to_string(peer_device) + " (no NVLink/P2P path)");
  cudaError_t e = cudaDeviceEnablePeerAccess(peer_device, 0);
  if (e == cudaErrorPeerAccessAlreadyEnabled) {
    (void)cudaGetLastError();
    e = cudaSuccess;
  }
  if (e != cudaSuccess) return fail_cuda(e, "cudaDeviceEnablePeerAccess");
  std::lock_guard<std::mutex> lk(m->mu);
  m->peers.insert(peer_device);
  return KVBM_OK;
  });
}

// base address + size of the cudaMalloc allocation containing p (driver entry point, no -lcuda needed)
static int allocation_range(uintptr_t p, uintptr_t* base, size_t* size)
{
  typedef int (*fn_t)(unsigned long long*, size_t*, unsigned long long);
  static fn_t fn = nullptr;
  if (!fn) {
    void* f = nullptr;
    cudaDriverEntryPointQueryResult q;
    cudaError_t e = cudaGetDriverEntryPoint("cuMemGetAddressRange", &f, cudaEnableDefault, &q);
    if (e != cudaSuccess || !f) return fail_cuda(e, "cudaGetDriverEntryPoint(cuMemGetAddressRange)");
    fn = reinterpret_cast<fn_t>(f);
  }
  unsigned long long b = 0;
  size_t s = 0;
  int r = fn(&b, &s, static_cast<unsigned long long>(p));
  if (r != 0) return fail(KVBM_ERR_CUDA, "cuMemGetAddressRange failed: " + std::to_string(r));
  *base = static_cast<uintptr_t>(b);
  *size = s;
  return KVBM_OK;
}

extern "C" int kvbm_manager_export_metadata(kvbm_transfer_manager* m, kvbm_layout_handle h, void* buf, size_t cap, size_t* len)
{
  return guarded([&]() -> int {
  if (!m || !len) return fail(KVBM_ERR, "null argument");
  std::lock_guard<std::mutex> lk(m->mu);
  Layout* L = m->find(h);
  if (!L) return fail(KVBM_ERR_HANDLE, "invalid handle");
  const size_t need = sizeof(BlobHeader) + L->allocs.size() * sizeof(BlobAlloc);
  *len = need;
  if (!buf) return KVBM_OK;
  if (cap < need) return fail(KVBM_ERR, "buffer too small for metadata");
  BlobHeader hd{};
  std::memcpy(hd.magic, kMagic, 8);
  hd.version = kBlobVersion;
  hd.fully_contiguous = L->fully_contiguous;
  hd.block_dim = static_cast<uint32_t>(L->block_dim);
  hd.storage = static_cast<uint32_t>(L->storage);
  hd.device_id = L->device_id;
  hd.n_allocs = static_cast<uint32_t>(L->allocs.size());
  hd.worker_id = m->worker_id;
  hd.pid = process_identity();
  const kvbm_layout_config& c = L->cfg;
  const uint64_t cfg[9] = {c.num_blocks, c.num_layers, c.outer_dim, c.page_size, c.inner_dim, c.alignment, c.dtype_width_bytes, c.num_heads,
                           static_cast<uint64_t>(c.allow_fp8 ? 1 : 0) | (static_cast<uint64_t>(L->kv_block_layout) << 8)};
  std::memcpy(hd.cfg, cfg, sizeof(cfg));
  auto* p = static_cast<unsigned char*>(buf);
  std::memcpy(p, &hd, sizeof(hd));
  p += sizeof(hd);
  DeviceGuard g(L->storage == KVBM_STORAGE_DEVICE ? L->device_id : -1);
  for (const Allocation& a : L->allocs) {
    BlobAlloc ba{};
    ba.addr = a.addr;
    ba.size = a.size;
    if (L->storage == KVBM_STORAGE_DEVICE && !L->remote) {
      uintptr_t base;
      size_t sz;
      int rc = allocation_range(a.addr, &base, &sz);
      if (rc) return rc;
      cudaIpcMemHandle_t ih;
      cudaError_t e = cudaIpcGetMemHandle(&ih, reinterpret_cast<void*>(base));
      if (e != cudaSuccess) return fail_cuda(e, "cudaIpcGetMemHandle");
      static_assert(sizeof(ih) == 64, "cudaIpcMemHandle_t is 64 bytes");
      std::memcpy(ba.ipc, &ih, 64);
      ba.has_ipc = 1;
      ba.offset_in_ipc = a.addr - base;
    }
    std::memcpy(p, &ba, sizeof(ba));
    p += sizeof(ba);
  }
  return KVBM_OK;
  });
}

static int import_metadata_impl(kvbm_transfer_manager* m, const void* buf, size_t len, const void* const* local_bases, size_t num_local_bases,
                                kvbm_layout_handle* out);

extern "C" int kvbm_manager_import_metadata(kvbm_transfer_manager* m, const void* buf, size_t len, kvbm_layout_handle* out)
{
  return guarded([&]() -> int {
  return import_metadata_impl(m, buf, len, nullptr, 0, out);
  });
}

// Host pools of another process that THIS process has mapped itself (POSIX / SysV shared memory, a hugetlbfs file, memory
// shared across fork): the importer names its own view of every allocation.  The CPU twin of the CUDA-IPC mapping above --
// what makes BASELINE configs[0] (two worker processes, CPU memcpy hand-off) a one-sided push like the NVLink path.
extern "C" int kvbm_manager_import_metadata_mapped(kvbm_transfer_manager* m, const void* buf, size_t len, const void* const* local_bases,
                                                   size_t num_local_bases, kvbm_layout_handle* out)
{
  return guarded([&]() -> int {
  if (!local_bases || num_local_bases == 0) return fail(KVBM_ERR, "local_bases: one address per allocation of the layout");
  return import_metadata_impl(m, buf, len, local_bases, num_local_bases, out);
  });
}

static int import_metadata_impl(kvbm_transfer_manager* m, const void* buf, size_t len, const void* const* local_bases, size_t num_local_bases,
                                kvbm_layout_handle* out)
{
  if (!m || !buf || !out) return fail(KVBM_ERR, "null argument");
  if (len < sizeof(BlobHeader)) return fail(KVBM_ERR, "metadata blob truncated");
  BlobHeader hd;
  std::memcpy(&hd, buf, sizeof(hd));
  if (std::memcmp(hd.magic, kMagic, 8) != 0) return fail(KVBM_ERR, "not a KVBM layout blob");
  if (hd.version != kBlobVersion)  // layout/serialize.rs version check
    return fail(KVBM_ERR_VERSION, "Unsupported layout descriptor version " + std::to_string(hd.version) + " (expected " + std::to_string(kBlobVersion) + ")");
  if (len < sizeof(BlobHeader) + hd.n_allocs * sizeof(BlobAlloc)) return fail(KVBM_ERR, "metadata blob truncated");
  kvbm_layout_config cfg{};
  cfg.num_blocks = hd.cfg[0];
  cfg.num_layers = hd.cfg[1];
  cfg.outer_dim = hd.cfg[2];
  cfg.page_size = hd.cfg[3];
  cfg.inner_dim = hd.cfg[4];
  cfg.alignment = hd.cfg[5];
  cfg.dtype_width_bytes = hd.cfg[6];
  cfg.num_heads = hd.cfg[7];
  cfg.allow_fp8 = static_cast<int>(hd.cfg[8] & 0xff);
  const bool same_process = hd.pid == process_identity();
  std::vector<uintptr_t> bases(hd.n_allocs);
  std::vector<size_t> sizes(hd.n_allocs);
  bool unmapped = false;
  const auto* pa = static_cast<const unsigned char*>(buf) + sizeof(BlobHeader);
  DeviceGuard g(m->device);
  for (uint32_t i = 0; i < hd.n_allocs; ++i) {
    BlobAlloc ba;
    std::memcpy(&ba, pa + i * sizeof(BlobAlloc), sizeof(ba));
    sizes[i] = ba.size;
    if (same_process) {
      bases[i] = ba.addr;  // same address space (peer access is enabled with kvbm_manager_enable_peer_access)
    } else if (!ba.has_ipc && local_bases) {
      if (hd.storage == KVBM_STORAGE_DEVICE) return fail(KVBM_ERR_UNSUPPORTED, "device allocations travel as CUDA IPC handles, not as caller-provided mappings");
      if (num_local_bases != hd.n_allocs)
        return fail(KVBM_ERR, "local_bases has " + std::to_string(num_local_bases) + " entries, the layout has " + std::to_string(hd.n_allocs) + " allocations");
      if (!local_bases[i]) return fail(KVBM_ERR, "null local mapping for allocation " + std::to_string(i));
      bases[i] = reinterpret_cast<uintptr_t>(local_bases[i]);  // this process's own mapping of the peer's shared memory
    } else if (!ba.has_ipc) {
      // Another process's System / Pinned pool (or device memory that could not be exported): its virtual addresses mean
      // nothing here.  The layout is registered as a DESCRIPTOR (geometry, handle, memory_region arithmetic) that no
      // transfer may touch -- the role NIXL's remote-descriptor-only entries play (manager/mod.rs:519-633).
      bases[i] = ba.addr;
      unmapped = true;
    } else {
      if (m->device < 0) return fail(KVBM_ERR_CUDA, "importing a device layout needs a CUDA manager");
      cudaIpcMemHandle_t ih;
      std::memcpy(&ih, ba.ipc, 64);
      const std::string key(reinterpret_cast<const char*>(ba.ipc), 64);
      void* mapped = nullptr;
      {
        std::lock_guard<std::mutex> lk(m->mu);
        auto it = m->ipc_cache.find(key);
        if (it != m->ipc_cache.end()) mapped = it->second;
      }
      if (!mapped) {
        cudaError_t e = cudaIpcOpenMemHandle(&mapped, ih, cudaIpcMemLazyEnablePeerAccess);
        if (e != cudaSuccess) return fail_cuda(e, "cudaIpcOpenMemHandle");
        cudaPointerAttributes pa{};
        const bool attr_ok = cudaPointerGetAttributes(&pa, mapped) == cudaSuccess;
        if (!attr_ok) (void)cudaGetLastError();
        std::lock_guard<std::mutex> lk(m->mu);
        m->ipc_cache[key] = mapped;
        if (attr_ok && pa.type == cudaMemoryTypeDevice && pa.device != m->device) m->peers.insert(pa.device);
      }
      bases[i] = reinterpret_cast<uintptr_t>(mapped) + ba.offset_in_ipc;
    }
  }
  Layout L;
  std::string why;
  int rc = hd.fully_contiguous ? make_fully_contiguous(cfg, bases.empty() ? 0 : bases[0], sizes.empty() ? 0 : sizes[0], &L, &why)
                               : make_layer_separate(cfg, bases.data(), sizes.data(), hd.n_allocs, static_cast<int>(hd.block_dim), &L, &why);
  if (rc) return fail(rc, why);
  L.remote = !same_process;
  L.unmapped = unmapped;
  L.kv_block_layout = static_cast<int>((hd.cfg[8] >> 8) & 0xff);
  return finish_register(m, std::move(L), static_cast<int>(hd.storage), hd.device_id, out);
}

// FullyContiguousLayoutBuilder::kv_block_layout / LayerSeparateLayoutBuilder::inner_shape (fully_contiguous.rs:83-88,
// layer_separate.rs:91-101): the format of one block of a registered layout; Unknown until set.
extern "C" int kvbm_manager_set_kv_block_layout(kvbm_transfer_manager* m, kvbm_layout_handle h, int kv_layout)
{
  return guarded([&]() -> int {
  if (!m) return fail(KVBM_ERR, "null manager");
  if (kv_layout < KVBM_KV_UNKNOWN || kv_layout > KVBM_KV_OPERATIONAL_NHD) return fail(KVBM_ERR, "unknown KvBlockLayout");
  std::lock_guard<std::mutex> lk(m->mu);
  Layout* L = m->find(h);
  if (!L) return fail(KVBM_ERR_HANDLE, "invalid layout handle");
  if (kv_layout != KVBM_KV_UNKNOWN) {
    // LayoutConfig::validate_for_kv_block_layout (config.rs:114-140); the head dimension is inner_dim / num_heads, the
    // figure consistent with required_bytes (:64-71) and with the chunk size K2 / K3 take
    int rc;
    if ((rc = need_num_heads(L->cfg)) || (rc = need_divisible_heads(L->cfg))) return rc;
    if ((kv_layout == KVBM_KV_UNIVERSAL_TP || kv_layout == KVBM_KV_UNIVERSAL_PP) && !L->fully_contiguous)
      return fail(KVBM_ERR_CONFIG, "universal KV block layouts exist only on fully contiguous layouts");  // layer_separate.rs:91-101
  }
  L->kv_block_layout = kv_layout;
  return KVBM_OK;
  });
}

extern "C" int kvbm_manager_kv_block_layout(kvbm_transfer_manager* m, kvbm_layout_handle h)
{
  if (!m) return -1;
  std::lock_guard<std::mutex> lk(m->mu);
  Layout* L = m->find(h);
  return L ? L->kv_block_layout : -1;
}

extern "C" int kvbm_select_transform_kernel(int src_kv_layout, int dst_kv_layout) { return select_transform_kernel(src_kv_layout, dst_kv_layout); }
extern "C" int kvbm_kv_layout_requires_transform(int a, int b) { return kv_requires_transform(a, b) ? 1 : 0; }

// kvbm_tp_reshard_plan's windows, after its checks, into *out.
static int tp_head_windows(size_t H, size_t src_tp, size_t dst_tp, size_t dst_rank, std::vector<kvbm_head_window>* out)
{
  if (!H || !src_tp || !dst_tp) return fail(KVBM_ERR_CONFIG, "num_kv_heads, src_tp and dst_tp must be positive");
  for (size_t tp : {src_tp, dst_tp})
    if (H % tp && tp % H)
      return fail(KVBM_ERR_CONFIG, std::to_string(H) + " KV heads cannot be sharded over TP " + std::to_string(tp) +
                                       ": one of the two must divide the other");
  if (dst_rank >= dst_tp) return fail(KVBM_ERR_RANGE, "dst_rank " + std::to_string(dst_rank) + " out of range for TP " + std::to_string(dst_tp));
  // vLLM's ownership: rank r of tp holds heads [r*H/tp, r*H/tp + max(1, H/tp)); replicated over tp/H ranks when tp > H
  const size_t d_first = dst_rank * H / dst_tp, d_count = std::max<size_t>(1, H / dst_tp);
  const size_t s_per = std::max<size_t>(1, H / src_tp), replicas = src_tp > H ? src_tp / H : 1;
  std::vector<kvbm_head_window>& w = *out;
  w.clear();
  for (size_t j = 0; j < d_count; ++j) {
    const size_t g = d_first + j;  // global head
    const size_t rank = replicas > 1 ? g * replicas + dst_rank % replicas : g / s_per;
    const size_t local = g - rank * H / src_tp;
    if (!w.empty() && w.back().src_rank == rank && w.back().src_head_begin + w.back().head_count == local)
      ++w.back().head_count;
    else
      w.push_back({rank, local, j, 1});
  }
  return KVBM_OK;
}

extern "C" int kvbm_tp_reshard_plan(size_t num_kv_heads, size_t src_tp, size_t dst_tp, size_t dst_rank, kvbm_head_window* out, size_t cap,
                                    size_t* n_out)
{
  if (!n_out) return fail(KVBM_ERR, "null argument");
  *n_out = 0;
  std::vector<kvbm_head_window> w;
  if (int rc = tp_head_windows(num_kv_heads, src_tp, dst_tp, dst_rank, &w)) return rc;
  *n_out = w.size();
  if (!out) return KVBM_OK;
  if (cap < w.size()) return fail(KVBM_ERR, "kvbm_tp_reshard_plan: " + std::to_string(w.size()) + " windows do not fit in " + std::to_string(cap));
  std::copy(w.begin(), w.end(), out);
  return KVBM_OK;
}

// The first layer of every stage of a pipeline of pp stages over L layers, and L at the end ([pp + 1] bounds): the partition's
// running sums, or an even split.  The library does not guess an engine's remainder policy, so an uneven L needs a partition.
static int stage_bounds(const char* side, size_t L, size_t pp, const size_t* parts, std::vector<size_t>* out)
{
  std::vector<size_t>& b = *out;
  b.assign(1, 0);
  if (!parts && L % pp)
    return fail(KVBM_ERR_CONFIG, std::string(side) + ": " + std::to_string(L) + " layers do not split evenly over PP " + std::to_string(pp) +
                                     "; pass the engine's stage layer counts");
  for (size_t p = 0; p < pp; ++p) {
    const size_t c = parts ? parts[p] : L / pp;
    if (c == 0) return fail(KVBM_ERR_CONFIG, std::string(side) + ": stage " + std::to_string(p) + " has no layers");
    b.push_back(b.back() + c);
  }
  if (b.back() != L)
    return fail(KVBM_ERR_CONFIG, std::string(side) + ": the stage layer counts sum to " + std::to_string(b.back()) + ", not num_layers " +
                                     std::to_string(L));
  return KVBM_OK;
}

// kvbm_tp_pp_reshard_plan's windows of decode rank dst_rank, after the checks every rank shares (the caller's), into *w.
static int tp_pp_windows(size_t num_kv_heads, size_t src_tp, size_t src_pp, const std::vector<size_t>& sb, size_t dst_tp,
                         const std::vector<size_t>& db, size_t dst_rank, std::vector<kvbm_shard_window>* w)
{
  std::vector<kvbm_head_window> heads;
  if (int rc = tp_head_windows(num_kv_heads, src_tp, dst_tp, dst_rank % dst_tp, &heads)) return rc;
  const size_t stage = dst_rank / dst_tp, d0 = db[stage], d1 = db[stage + 1];
  w->clear();
  for (size_t p = 0; p < src_pp; ++p) {
    const size_t lo = std::max(d0, sb[p]), hi = std::min(d1, sb[p + 1]);
    if (lo >= hi) continue;
    for (const kvbm_head_window& h : heads)
      w->push_back({p * src_tp + h.src_rank, lo - sb[p], lo - d0, hi - lo, h.src_head_begin, h.dst_head_begin, h.head_count});
  }
  return KVBM_OK;
}

// The checks both PP x TP plans make before they name a rank: positive arguments and each side's stage bounds.
static int tp_pp_bounds(size_t num_kv_heads, size_t num_layers, size_t src_tp, size_t src_pp, const size_t* src_stage_layers, size_t dst_tp,
                        size_t dst_pp, const size_t* dst_stage_layers, std::vector<size_t>* sb, std::vector<size_t>* db)
{
  if (!num_kv_heads || !num_layers || !src_tp || !src_pp || !dst_tp || !dst_pp)
    return fail(KVBM_ERR_CONFIG, "num_kv_heads, num_layers and every TP and PP degree must be positive");
  int rc;
  if ((rc = stage_bounds("source", num_layers, src_pp, src_stage_layers, sb)) || (rc = stage_bounds("destination", num_layers, dst_pp, dst_stage_layers, db)))
    return rc;
  return KVBM_OK;
}

extern "C" int kvbm_tp_pp_reshard_plan(size_t num_kv_heads, size_t num_layers, size_t src_tp, size_t src_pp, const size_t* src_stage_layers,
                                       size_t dst_tp, size_t dst_pp, const size_t* dst_stage_layers, size_t dst_rank, kvbm_shard_window* out,
                                       size_t cap, size_t* n_out)
{
  return guarded([&]() -> int {
  if (!n_out) return fail(KVBM_ERR, "null argument");
  *n_out = 0;
  std::vector<size_t> sb, db;
  int rc;
  if ((rc = tp_pp_bounds(num_kv_heads, num_layers, src_tp, src_pp, src_stage_layers, dst_tp, dst_pp, dst_stage_layers, &sb, &db))) return rc;
  if (dst_rank >= dst_pp * dst_tp)
    return fail(KVBM_ERR_RANGE, "dst_rank " + std::to_string(dst_rank) + " out of range for PP " + std::to_string(dst_pp) + " x TP " +
                                    std::to_string(dst_tp));
  std::vector<kvbm_shard_window> w;
  if ((rc = tp_pp_windows(num_kv_heads, src_tp, src_pp, sb, dst_tp, db, dst_rank, &w))) return rc;
  *n_out = w.size();
  if (!out) return KVBM_OK;
  if (cap < w.size()) return fail(KVBM_ERR, "kvbm_tp_pp_reshard_plan: " + std::to_string(w.size()) + " windows do not fit in " + std::to_string(cap));
  std::copy(w.begin(), w.end(), out);
  return KVBM_OK;
  });
}

extern "C" int kvbm_tp_pp_scatter_plan(size_t num_kv_heads, size_t num_layers, size_t src_tp, size_t src_pp, const size_t* src_stage_layers,
                                       size_t dst_tp, size_t dst_pp, const size_t* dst_stage_layers, size_t src_rank, kvbm_scatter_window* out,
                                       size_t cap, size_t* n_out)
{
  return guarded([&]() -> int {
  if (!n_out) return fail(KVBM_ERR, "null argument");
  *n_out = 0;
  std::vector<size_t> sb, db;
  int rc;
  if ((rc = tp_pp_bounds(num_kv_heads, num_layers, src_tp, src_pp, src_stage_layers, dst_tp, dst_pp, dst_stage_layers, &sb, &db))) return rc;
  if (src_rank >= src_pp * src_tp)
    return fail(KVBM_ERR_RANGE, "src_rank " + std::to_string(src_rank) + " out of range for PP " + std::to_string(src_pp) + " x TP " +
                                    std::to_string(src_tp));
  // the inverse of the gather plans: every decode rank's windows that read src_rank, in ascending decode rank
  std::vector<kvbm_scatter_window> w;
  std::vector<kvbm_shard_window> g;
  for (size_t d = 0; d < dst_pp * dst_tp; ++d) {
    if ((rc = tp_pp_windows(num_kv_heads, src_tp, src_pp, sb, dst_tp, db, d, &g))) return rc;
    for (const kvbm_shard_window& x : g)
      if (x.src_rank == src_rank)
        w.push_back({d, x.src_layer_begin, x.dst_layer_begin, x.layer_count, x.src_head_begin, x.dst_head_begin, x.head_count});
  }
  *n_out = w.size();
  if (!out) return KVBM_OK;
  if (cap < w.size()) return fail(KVBM_ERR, "kvbm_tp_pp_scatter_plan: " + std::to_string(w.size()) + " windows do not fit in " + std::to_string(cap));
  std::copy(w.begin(), w.end(), out);
  return KVBM_OK;
  });
}

extern "C" int kvbm_manager_set_capabilities(kvbm_transfer_manager* m, const kvbm_transfer_capabilities* caps)
{
  if (!m || !caps) return fail(KVBM_ERR, "null argument");
  std::lock_guard<std::mutex> lk(m->mu);
  m->caps = *caps;
  return KVBM_OK;
}

extern "C" int kvbm_manager_execute_transfer(kvbm_transfer_manager* m, kvbm_layout_handle src, const size_t* src_ids, kvbm_layout_handle dst,
                                             const size_t* dst_ids, size_t n, const kvbm_transfer_options* opts, kvbm_notification* out)
{
  return guarded([&]() -> int {
  if (!m) return fail(KVBM_ERR, "null manager");
  const size_t* s[1] = {src_ids};
  const size_t* d[1] = {dst_ids};
  return execute(m, src, 1, &dst, s, d, n, true, opts, out);
  });
}

extern "C" int kvbm_manager_execute_gather(kvbm_transfer_manager* m, size_t num_srcs, const kvbm_layout_handle* srcs,
                                           const size_t* const* src_ids, kvbm_layout_handle dst, const size_t* dst_ids, size_t n,
                                           const kvbm_head_window* windows, size_t num_windows, const kvbm_transfer_options* opts,
                                           kvbm_notification* out)
{
  return guarded([&]() -> int {
  if (!m) return fail(KVBM_ERR, "null manager");
  return execute_gather(m, num_srcs, srcs, src_ids, dst, dst_ids, n, windows, num_windows, opts, out);
  });
}

extern "C" int kvbm_manager_execute_repage(kvbm_transfer_manager* m, kvbm_layout_handle src, const size_t* src_ids, size_t n_src,
                                           kvbm_layout_handle dst, const size_t* dst_ids, size_t n_dst, size_t token_begin, size_t token_end,
                                           const kvbm_transfer_options* opts, kvbm_notification* out)
{
  return guarded([&]() -> int {
  if (!m) return fail(KVBM_ERR, "null manager");
  const kvbm_repage_batch_seq q{token_begin, token_end, &src_ids, n_src, dst_ids, n_dst};
  return execute_repage(m, 1, &src, dst, &q, 1, /*windows=*/nullptr, 1, opts, out, /*ls=*/nullptr, /*gather=*/false);
  });
}

extern "C" int kvbm_manager_execute_repage_gather(kvbm_transfer_manager* m, size_t num_srcs, const kvbm_layout_handle* srcs,
                                                  const size_t* const* src_ids, size_t n_src, kvbm_layout_handle dst, const size_t* dst_ids,
                                                  size_t n_dst, size_t token_begin, size_t token_end, const kvbm_head_window* windows,
                                                  size_t num_windows, const kvbm_transfer_options* opts, kvbm_notification* out)
{
  return guarded([&]() -> int {
  if (!m) return fail(KVBM_ERR, "null manager");
  const kvbm_repage_batch_seq q{token_begin, token_end, src_ids, n_src, dst_ids, n_dst};
  return execute_repage(m, num_srcs, srcs, dst, &q, 1, windows, num_windows, opts, out);
  });
}

extern "C" int kvbm_manager_execute_repage_scatter(kvbm_transfer_manager* m, kvbm_layout_handle src, const size_t* src_ids, size_t n_src,
                                                   size_t num_dsts, const kvbm_layout_handle* dsts, const size_t* const* dst_ids, size_t n_dst,
                                                   size_t token_begin, size_t token_end, const kvbm_scatter_window* windows,
                                                   size_t num_windows, const kvbm_transfer_options* opts, kvbm_notification* out)
{
  return guarded([&]() -> int {
  if (!m) return fail(KVBM_ERR, "null manager");
  const kvbm_scatter_batch_seq q{token_begin, token_end, src_ids, n_src, dst_ids, n_dst};
  return execute_repage_scatter(m, src, num_dsts, dsts, &q, 1, windows, num_windows, opts, out);
  });
}

// The start of every entry that may stream: a null manager, then the layer stream's shape when there is one or `streamed`
// requires it.
static int stream_entry(kvbm_transfer_manager* m, const kvbm_layer_stream* ls, size_t num_srcs, bool streamed, kvbm_notification* out)
{
  if (!m) return fail(KVBM_ERR, "null manager");
  if (out) *out = 0;
  return ls || streamed ? check_layer_stream_shape(ls, num_srcs) : KVBM_OK;
}

extern "C" int kvbm_manager_execute_repage_scatter_streamed(kvbm_transfer_manager* m, kvbm_layout_handle src, const size_t* src_ids,
                                                            size_t n_src, size_t num_dsts, const kvbm_layout_handle* dsts,
                                                            const size_t* const* dst_ids, size_t n_dst, size_t token_begin, size_t token_end,
                                                            const kvbm_scatter_window* windows, size_t num_windows, const kvbm_layer_stream* ls,
                                                            const kvbm_transfer_options* opts, kvbm_notification* out)
{
  return guarded([&]() -> int {
  if (int rc = stream_entry(m, ls, 1, true, out)) return rc;
  const kvbm_scatter_batch_seq q{token_begin, token_end, src_ids, n_src, dst_ids, n_dst};
  return execute_repage_scatter(m, src, num_dsts, dsts, &q, 1, windows, num_windows, opts, out, ls);
  });
}

extern "C" int kvbm_manager_execute_repage_scatter_batch(kvbm_transfer_manager* m, kvbm_layout_handle src, size_t num_dsts,
                                                         const kvbm_layout_handle* dsts, const kvbm_scatter_batch_seq* seqs, size_t num_seqs,
                                                         const kvbm_scatter_window* windows, size_t num_windows, const kvbm_layer_stream* ls,
                                                         const kvbm_transfer_options* opts, kvbm_notification* out)
{
  return guarded([&]() -> int {
  if (int rc = stream_entry(m, ls, 1, false, out)) return rc;
  return execute_repage_scatter(m, src, num_dsts, dsts, seqs, num_seqs, windows, num_windows, opts, out, ls, kSeqs);
  });
}

extern "C" int kvbm_manager_execute_repage_scatter_anypage(kvbm_transfer_manager* m, kvbm_layout_handle src, size_t num_dsts,
                                                           const kvbm_layout_handle* dsts, const kvbm_scatter_batch_seq* seqs, size_t num_seqs,
                                                           const kvbm_scatter_window* windows, size_t num_windows, const kvbm_layer_stream* ls,
                                                           const kvbm_transfer_options* opts, kvbm_notification* out)
{
  return guarded([&]() -> int {
  if (int rc = stream_entry(m, ls, 1, false, out)) return rc;
  return execute_repage_scatter(m, src, num_dsts, dsts, seqs, num_seqs, windows, num_windows, opts, out, ls, kPhased);
  });
}

// The body of kvbm_manager_execute_repage_scatter_routed (units kRouted) and kvbm_manager_execute_repage_scatter_routed_anypage
// (kRoutedPhased).
static int execute_repage_scatter_routed(kvbm_transfer_manager* m, kvbm_layout_handle src, size_t num_dsts, const kvbm_layout_handle* dsts,
                                         const kvbm_scatter_route_seq* seqs, size_t num_seqs, const kvbm_scatter_window* windows,
                                         size_t num_windows, const kvbm_layer_stream* ls, const kvbm_transfer_options* opts,
                                         kvbm_notification* out, RepageUnits units)
{
  return guarded([&]() -> int {
  if (int rc = stream_entry(m, ls, 1, false, out)) return rc;
  std::vector<kvbm_scatter_batch_seq> qs(seqs ? num_seqs : 0);
  std::vector<uint32_t> masks(std::max<size_t>(1, qs.size()));  // never empty: a null masks is an unrouted call
  for (size_t i = 0; i < qs.size(); ++i) {
    const kvbm_scatter_route_seq& s = seqs[i];
    qs[i] = kvbm_scatter_batch_seq{s.token_begin, s.token_end, s.src_ids, s.n_src, s.dst_ids, s.n_dst};
    masks[i] = s.dst_mask;
  }
  return execute_repage_scatter(m, src, num_dsts, dsts, seqs ? qs.data() : nullptr, num_seqs, windows, num_windows, opts, out, ls, units,
                                masks.data());
  });
}

extern "C" int kvbm_manager_execute_repage_scatter_routed(kvbm_transfer_manager* m, kvbm_layout_handle src, size_t num_dsts,
                                                          const kvbm_layout_handle* dsts, const kvbm_scatter_route_seq* seqs, size_t num_seqs,
                                                          const kvbm_scatter_window* windows, size_t num_windows, const kvbm_layer_stream* ls,
                                                          const kvbm_transfer_options* opts, kvbm_notification* out)
{
  return execute_repage_scatter_routed(m, src, num_dsts, dsts, seqs, num_seqs, windows, num_windows, ls, opts, out, kRouted);
}

extern "C" int kvbm_manager_execute_repage_scatter_routed_anypage(kvbm_transfer_manager* m, kvbm_layout_handle src, size_t num_dsts,
                                                                  const kvbm_layout_handle* dsts, const kvbm_scatter_route_seq* seqs,
                                                                  size_t num_seqs, const kvbm_scatter_window* windows, size_t num_windows,
                                                                  const kvbm_layer_stream* ls, const kvbm_transfer_options* opts,
                                                                  kvbm_notification* out)
{
  return execute_repage_scatter_routed(m, src, num_dsts, dsts, seqs, num_seqs, windows, num_windows, ls, opts, out, kRoutedPhased);
}

// The head windows of a staged plan's windows, in hw[], or null without windows.  Only the first KVBM_GATHER_MAX_SOURCES are
// copied: check_gather_windows rejects more windows than that before it reads any.
static const kvbm_head_window* head_windows(const kvbm_shard_window* windows, size_t nw, kvbm_head_window* hw)
{
  if (!windows) return nullptr;
  for (size_t j = 0; j < std::min<size_t>(nw, KVBM_GATHER_MAX_SOURCES); ++j)
    hw[j] = kvbm_head_window{windows[j].src_rank, windows[j].src_head_begin, windows[j].dst_head_begin, windows[j].head_count};
  return hw;
}

extern "C" int kvbm_manager_execute_gather_streamed(kvbm_transfer_manager* m, size_t num_srcs, const kvbm_layout_handle* srcs,
                                                    const size_t* const* src_ids, kvbm_layout_handle dst, const size_t* dst_ids, size_t n,
                                                    const kvbm_head_window* windows, size_t num_windows, const kvbm_layer_stream* ls,
                                                    const kvbm_transfer_options* opts, kvbm_notification* out)
{
  return guarded([&]() -> int {
  if (int rc = stream_entry(m, ls, num_srcs, true, out)) return rc;
  return execute_gather(m, num_srcs, srcs, src_ids, dst, dst_ids, n, windows, num_windows, opts, out, ls);
  });
}

extern "C" int kvbm_manager_execute_stage_gather(kvbm_transfer_manager* m, size_t num_srcs, const kvbm_layout_handle* srcs,
                                                 const size_t* const* src_ids, kvbm_layout_handle dst, const size_t* dst_ids, size_t n,
                                                 const kvbm_shard_window* windows, size_t num_windows, const kvbm_layer_stream* ls,
                                                 const kvbm_transfer_options* opts, kvbm_notification* out)
{
  return guarded([&]() -> int {
  if (int rc = stream_entry(m, ls, num_srcs, false, out)) return rc;
  kvbm_head_window hw[KVBM_GATHER_MAX_SOURCES];
  return execute_gather(m, num_srcs, srcs, src_ids, dst, dst_ids, n, head_windows(windows, num_windows, hw), num_windows, opts, out, ls, windows);
  });
}

extern "C" int kvbm_manager_execute_stage_repage_gather(kvbm_transfer_manager* m, size_t num_srcs, const kvbm_layout_handle* srcs,
                                                        const size_t* const* src_ids, size_t n_src, kvbm_layout_handle dst,
                                                        const size_t* dst_ids, size_t n_dst, size_t token_begin, size_t token_end,
                                                        const kvbm_shard_window* windows, size_t num_windows, const kvbm_layer_stream* ls,
                                                        const kvbm_transfer_options* opts, kvbm_notification* out)
{
  return guarded([&]() -> int {
  if (int rc = stream_entry(m, ls, num_srcs, false, out)) return rc;
  kvbm_head_window hw[KVBM_GATHER_MAX_SOURCES];
  const kvbm_repage_batch_seq q{token_begin, token_end, src_ids, n_src, dst_ids, n_dst};
  return execute_repage(m, num_srcs, srcs, dst, &q, 1, head_windows(windows, num_windows, hw), num_windows, opts, out, ls, /*gather=*/true,
                        windows);
  });
}

extern "C" int kvbm_manager_execute_repage_batch(kvbm_transfer_manager* m, size_t num_srcs, const kvbm_layout_handle* srcs,
                                                 kvbm_layout_handle dst, const kvbm_repage_batch_seq* seqs, size_t num_seqs,
                                                 const kvbm_shard_window* windows, size_t num_windows, const kvbm_layer_stream* ls,
                                                 const kvbm_transfer_options* opts, kvbm_notification* out)
{
  return guarded([&]() -> int {
  if (int rc = stream_entry(m, ls, num_srcs, false, out)) return rc;
  kvbm_head_window hw[KVBM_GATHER_MAX_SOURCES];
  return execute_repage(m, num_srcs, srcs, dst, seqs, num_seqs, head_windows(windows, num_windows, hw), num_windows, opts, out, ls,
                        /*gather=*/true, windows, kSeqs);
  });
}

extern "C" int kvbm_manager_execute_repage_anypage(kvbm_transfer_manager* m, size_t num_srcs, const kvbm_layout_handle* srcs,
                                                   kvbm_layout_handle dst, const kvbm_repage_batch_seq* seqs, size_t num_seqs,
                                                   const kvbm_shard_window* windows, size_t num_windows, const kvbm_layer_stream* ls,
                                                   const kvbm_transfer_options* opts, kvbm_notification* out)
{
  return guarded([&]() -> int {
  if (int rc = stream_entry(m, ls, num_srcs, false, out)) return rc;
  kvbm_head_window hw[KVBM_GATHER_MAX_SOURCES];
  return execute_repage(m, num_srcs, srcs, dst, seqs, num_seqs, head_windows(windows, num_windows, hw), num_windows, opts, out, ls,
                        /*gather=*/true, windows, kPhased);
  });
}

// The body of kvbm_manager_execute_repage_batch_routed (units kRouted) and kvbm_manager_execute_repage_batch_routed_anypage
// (kRoutedPhased).
static int execute_repage_batch_routed(kvbm_transfer_manager* m, size_t num_srcs, const kvbm_layout_handle* srcs, kvbm_layout_handle dst,
                                       const kvbm_repage_route_seq* seqs, size_t num_seqs, const kvbm_shard_window* windows,
                                       size_t num_windows, const kvbm_layer_stream* ls, const kvbm_transfer_options* opts,
                                       kvbm_notification* out, RepageUnits units)
{
  return guarded([&]() -> int {
  if (int rc = stream_entry(m, ls, num_srcs, false, out)) return rc;
  kvbm_head_window hw[KVBM_GATHER_MAX_SOURCES];
  std::vector<kvbm_repage_batch_seq> qs(seqs ? num_seqs : 0);
  std::vector<uint32_t> masks(std::max<size_t>(1, qs.size()));  // never empty: a null masks is an unrouted call
  for (size_t i = 0; i < qs.size(); ++i) {
    const kvbm_repage_route_seq& s = seqs[i];
    qs[i] = kvbm_repage_batch_seq{s.token_begin, s.token_end, s.src_ids, s.n_src, s.dst_ids, s.n_dst};
    masks[i] = s.src_mask;
  }
  return execute_repage(m, num_srcs, srcs, dst, seqs ? qs.data() : nullptr, num_seqs, head_windows(windows, num_windows, hw), num_windows,
                        opts, out, ls, /*gather=*/true, windows, units, masks.data());
  });
}

extern "C" int kvbm_manager_execute_repage_batch_routed(kvbm_transfer_manager* m, size_t num_srcs, const kvbm_layout_handle* srcs,
                                                        kvbm_layout_handle dst, const kvbm_repage_route_seq* seqs, size_t num_seqs,
                                                        const kvbm_shard_window* windows, size_t num_windows, const kvbm_layer_stream* ls,
                                                        const kvbm_transfer_options* opts, kvbm_notification* out)
{
  return execute_repage_batch_routed(m, num_srcs, srcs, dst, seqs, num_seqs, windows, num_windows, ls, opts, out, kRouted);
}

extern "C" int kvbm_manager_execute_repage_batch_routed_anypage(kvbm_transfer_manager* m, size_t num_srcs, const kvbm_layout_handle* srcs,
                                                                kvbm_layout_handle dst, const kvbm_repage_route_seq* seqs, size_t num_seqs,
                                                                const kvbm_shard_window* windows, size_t num_windows,
                                                                const kvbm_layer_stream* ls, const kvbm_transfer_options* opts,
                                                                kvbm_notification* out)
{
  return execute_repage_batch_routed(m, num_srcs, srcs, dst, seqs, num_seqs, windows, num_windows, ls, opts, out, kRoutedPhased);
}

extern "C" int kvbm_manager_execute_repage_gather_streamed(kvbm_transfer_manager* m, size_t num_srcs, const kvbm_layout_handle* srcs,
                                                           const size_t* const* src_ids, size_t n_src, kvbm_layout_handle dst,
                                                           const size_t* dst_ids, size_t n_dst, size_t token_begin, size_t token_end,
                                                           const kvbm_head_window* windows, size_t num_windows, const kvbm_layer_stream* ls,
                                                           const kvbm_transfer_options* opts, kvbm_notification* out)
{
  return guarded([&]() -> int {
  if (int rc = stream_entry(m, ls, num_srcs, true, out)) return rc;
  const kvbm_repage_batch_seq q{token_begin, token_end, src_ids, n_src, dst_ids, n_dst};
  return execute_repage(m, num_srcs, srcs, dst, &q, 1, windows, num_windows, opts, out, ls);
  });
}

extern "C" int kvbm_manager_execute_fanout(kvbm_transfer_manager* m, kvbm_layout_handle src, int num_dsts, const kvbm_layout_handle* dsts,
                                           const size_t* const* src_ids, const size_t* const* dst_ids, size_t n, int replicate,
                                           const kvbm_transfer_options* opts, kvbm_notification* out)
{
  return guarded([&]() -> int {
  if (!m || !dsts) return fail(KVBM_ERR, "null argument");
  bool rep = replicate != 0;
  if (!rep && src_ids) {
    rep = true;
    for (int d = 1; d < num_dsts; ++d)
      if (src_ids[d] != src_ids[0]) rep = false;
  }
  return execute(m, src, num_dsts, dsts, src_ids, dst_ids, n, rep, opts, out);
  });
}

extern "C" int kvbm_notification_is_complete(kvbm_transfer_manager* m, kvbm_notification n)
{
  if (!m) return -1;
  if (n == 0) return 1;
  // Lock-free against execute() recycling the slot: the owner word is atomic, the completion word lives at a fixed
  // address for the manager's lifetime, and the owner is re-checked after the completion word was read.
  Slot& sl = m->slots[(n - 1) % kSlots];
  const uint64_t s1 = sl.seq.load(std::memory_order_acquire);
  if (s1 != n) return s1 > n ? 1 : -1;  // slot recycled by a later transfer => ours completed
  const uint32_t v = __atomic_load_n(sl.host_flag, __ATOMIC_ACQUIRE);
  if (sl.seq.load(std::memory_order_acquire) != n) return 1;
  if (v == 0xFFFFFFFFu) return -2;  // the gated kernel gave up waiting for a layer_ready flag
  return v == static_cast<uint32_t>(n) ? 1 : 0;
}

extern "C" int kvbm_notification_wait(kvbm_transfer_manager* m, kvbm_notification n, int64_t timeout_us)
{
  return guarded([&]() -> int {
  if (!m) return fail(KVBM_ERR, "null manager");
  const auto t0 = std::chrono::steady_clock::now();
  unsigned spins = 0;
  for (;;) {
    int c = kvbm_notification_is_complete(m, n);
    if (c == 1) return KVBM_OK;
    if (c == -2) return fail(KVBM_ERR_TIMEOUT, "gated transfer aborted: a layer_ready flag was not released within the gate timeout");
    if (c < 0) return fail(KVBM_ERR_HANDLE, "unknown notification");
    if ((++spins & 63) == 0) {
      if (timeout_us >= 0 &&
          std::chrono::duration_cast<std::chrono::microseconds>(std::chrono::steady_clock::now() - t0).count() > timeout_us)
        return fail(KVBM_ERR_TIMEOUT, "transfer did not complete in time");
      sched_yield();
    }
  }
  });
}

extern "C" uint64_t kvbm_manager_bytes_moved(kvbm_transfer_manager* m) { return m ? m->bytes_moved.load() : 0; }
extern "C" uint64_t kvbm_manager_h2d_bytes(kvbm_transfer_manager* m) { return m ? m->h2d_bytes.load() : 0; }

// =====================================================================================================
// SerializedLayout / LayoutDescriptor in the reference's wire formats (SURVEY.md 8 f3); codec in serialized_layout.hpp
// =====================================================================================================
namespace kvbm_host {

static const char kTransportMagic[8] = {'K', 'V', 'B', 'M', 'I', 'P', 'C', '1'};

static std::string agent_name_of(uint64_t worker_id) { return "kvbm-b200-ipc-" + std::to_string(worker_id); }

// PhysicalLayout::to_descriptor (layout/physical.rs:163-187)
static kvbm_wire::Descriptor to_wire(const Layout& L, const std::string& agent)
{
  kvbm_wire::Descriptor d;
  d.version = 1;
  d.num_blocks = L.cfg.num_blocks;
  d.num_layers = L.cfg.num_layers;
  d.outer_dim = L.cfg.outer_dim;
  d.page_size = L.cfg.page_size;
  d.inner_dim = L.cfg.inner_dim;
  d.alignment = L.cfg.alignment == 0 ? 1 : L.cfg.alignment;
  d.dtype_width_bytes = L.cfg.dtype_width_bytes;
  d.has_num_heads = L.cfg.num_heads != 0;
  d.num_heads = L.cfg.num_heads;
  switch (L.storage) {
    case KVBM_STORAGE_PINNED: d.location = kvbm_wire::kPinned; break;
    case KVBM_STORAGE_DEVICE:
      d.location = kvbm_wire::kDevice;
      d.location_arg = static_cast<uint64_t>(L.device_id);
      break;
    case KVBM_STORAGE_DISK: d.location = kvbm_wire::kDisk; break;
    default: d.location = kvbm_wire::kSystem;
  }
  d.agent_name = agent;
  d.mem_type = L.storage == KVBM_STORAGE_DEVICE ? kvbm_wire::kVram : L.storage == KVBM_STORAGE_DISK ? kvbm_wire::kFile : kvbm_wire::kDram;
  d.nixl_device_id = L.storage == KVBM_STORAGE_DEVICE ? static_cast<uint64_t>(L.device_id) : 0;
  for (const Allocation& a : L.allocs) d.regions.push_back({a.addr, a.size});
  d.fully_contiguous = L.fully_contiguous;
  d.block_dim = L.block_dim == KVBM_BLOCK_IS_SECOND_DIM ? 1u : 0u;
  d.kv_block_layout = L.kv_block_layout >= KVBM_KV_UNIVERSAL_TP && L.kv_block_layout <= KVBM_KV_CUSTOM ? static_cast<uint32_t>(L.kv_block_layout - 1) : kvbm_wire::kKvUnknown;
  return d;
}

static kvbm_layout_config config_of(const kvbm_wire::Descriptor& d)
{
  kvbm_layout_config c{};
  c.num_blocks = d.num_blocks;
  c.num_layers = d.num_layers;
  c.outer_dim = d.outer_dim;
  c.page_size = d.page_size;
  c.inner_dim = d.inner_dim;
  c.alignment = d.alignment;
  c.dtype_width_bytes = d.dtype_width_bytes;
  c.num_heads = d.has_num_heads ? d.num_heads : 0;
  c.allow_fp8 = d.dtype_width_bytes == 1;
  return c;
}

// the structural checks of PhysicalLayout::from_descriptor (layout/physical.rs:203-262)
static int check_descriptor(const kvbm_wire::Descriptor& d)
{
  if (d.version > 1) return fail(KVBM_ERR_VERSION, "Unsupported serialization version: " + std::to_string(d.version) + ". Maximum supported: 1");
  if (d.fully_contiguous && d.regions.size() != 1)
    return fail(KVBM_ERR_CONFIG, "FullyContiguous layout requires exactly 1 memory region, got " + std::to_string(d.regions.size()));
  if (!d.fully_contiguous && d.regions.size() != d.num_layers)
    return fail(KVBM_ERR_CONFIG, "LayerSeparate layout requires " + std::to_string(d.num_layers) + " memory regions (one per layer), got " +
                                     std::to_string(d.regions.size()));
  return KVBM_OK;
}

static int copy_out(const void* data, size_t need, void* buf, size_t cap, size_t* len)
{
  *len = need;
  if (!buf) return KVBM_OK;
  if (cap < need) return fail(KVBM_ERR, "buffer too small");
  std::memcpy(buf, data, need);
  return KVBM_OK;
}

}  // namespace kvbm_host

extern "C" int kvbm_layout_descriptor_json(kvbm_transfer_manager* m, kvbm_layout_handle h, char* buf, size_t cap, size_t* len)
{
  return guarded([&]() -> int {
  if (!m || !len) return fail(KVBM_ERR, "null argument");
  std::string js;
  {
    std::lock_guard<std::mutex> lk(m->mu);
    Layout* L = m->find(h);
    if (!L) return fail(KVBM_ERR_HANDLE, "invalid handle");
    js = kvbm_wire::descriptor_to_json(to_wire(*L, agent_name_of(m->worker_id)));
  }
  return copy_out(js.data(), js.size(), buf, cap, len);
  });
}

extern "C" int kvbm_manager_import_descriptor_json(kvbm_transfer_manager* m, const char* json, size_t len, kvbm_layout_handle* out)
{
  return guarded([&]() -> int {
  if (!m || !json || !out) return fail(KVBM_ERR, "null argument");
  kvbm_wire::Descriptor d;
  std::string why;
  if (!kvbm_wire::descriptor_from_json(json, len, &d, &why)) return fail(KVBM_ERR, why);
  int rc = check_descriptor(d);
  if (rc) return rc;
  const kvbm_layout_config cfg = config_of(d);
  Layout L;
  if (d.fully_contiguous) {
    rc = make_fully_contiguous(cfg, static_cast<uintptr_t>(d.regions[0].addr), d.regions[0].size, &L, &why);
  } else {
    std::vector<uintptr_t> bases;
    std::vector<size_t> sizes;
    for (const auto& g : d.regions) {
      bases.push_back(static_cast<uintptr_t>(g.addr));
      sizes.push_back(g.size);
    }
    rc = make_layer_separate(cfg, bases.data(), sizes.data(), bases.size(), d.block_dim ? KVBM_BLOCK_IS_SECOND_DIM : KVBM_BLOCK_IS_FIRST_DIM, &L, &why);
  }
  if (rc) return fail(rc, why);
  L.kv_block_layout = d.kv_block_layout <= kvbm_wire::kCustom ? static_cast<int>(d.kv_block_layout) + 1 : KVBM_KV_UNKNOWN;
  const int storage = d.location == kvbm_wire::kDevice ? KVBM_STORAGE_DEVICE
                      : d.location == kvbm_wire::kPinned ? KVBM_STORAGE_PINNED
                      : d.location == kvbm_wire::kDisk   ? KVBM_STORAGE_DISK
                                                         : KVBM_STORAGE_SYSTEM;
  return finish_register(m, std::move(L), storage, d.location == kvbm_wire::kDevice ? static_cast<int>(d.location_arg) : 0, out);
  });
}

// TransferManager::export_metadata (manager/mod.rs:112, registry :519-556): every local host / device layout, one blob.
// `nixl_metadata` carries this library's transport records instead of a NIXL agent's: per layout one KVBMLAY1 blob with a
// CUDA IPC handle per allocation, so the importing process can map the pools and reach them over NVLink.
extern "C" int kvbm_manager_export_serialized_layout(kvbm_transfer_manager* m, void* buf, size_t cap, size_t* len)
{
  return guarded([&]() -> int {
  if (!m || !len) return fail(KVBM_ERR, "null argument");
  std::vector<kvbm_layout_handle> handles;
  kvbm_wire::Bundle b;
  b.worker_id = m->worker_id;
  b.agent_name = agent_name_of(m->worker_id);
  {
    std::lock_guard<std::mutex> lk(m->mu);
    for (auto& kv : m->layouts)
      if (!kv.second->remote && kv.second->storage != KVBM_STORAGE_DISK) handles.push_back(kv.first);
    std::sort(handles.begin(), handles.end());
    for (kvbm_layout_handle h : handles) {
      kvbm_wire::Logical l;
      l.worker_id = m->worker_id;
      l.layout_id = static_cast<uint16_t>(h & 0xffff);
      l.logical_type = kvbm_wire::kG2;  // LocalLayoutDescriptor::new_with_default_type (manager/metadata.rs:70-76)
      l.layout = to_wire(*m->find(h), b.agent_name);
      b.layouts.push_back(std::move(l));
    }
  }
  kvbm_wire::Writer t;
  t.raw(kTransportMagic, 8);
  t.le(handles.size(), 4);
  for (kvbm_layout_handle h : handles) {
    size_t need = 0;
    int rc = kvbm_manager_export_metadata(m, h, nullptr, 0, &need);
    if (rc) return rc;
    std::vector<uint8_t> one(need);
    rc = kvbm_manager_export_metadata(m, h, one.data(), one.size(), &need);
    if (rc) return rc;
    t.le(one.size(), 4);
    t.raw(one.data(), one.size());
  }
  b.nixl_metadata = std::move(t.out);
  const std::vector<uint8_t> bytes = kvbm_wire::encode_bundle(b);
  return copy_out(bytes.data(), bytes.size(), buf, cap, len);
  });
}

// TransferManager::import_metadata (manager/mod.rs:130, registry :572-633)
extern "C" int kvbm_manager_import_serialized_layout(kvbm_transfer_manager* m, const void* buf, size_t len, kvbm_layout_handle* out, size_t cap,
                                                     size_t* n_out)
{
  return guarded([&]() -> int {
  if (!m || !buf || !n_out) return fail(KVBM_ERR, "null argument");
  kvbm_wire::Bundle b;
  std::string why;
  if (!kvbm_wire::decode_bundle(buf, len, &b, &why)) return fail(KVBM_ERR, why);
  const auto key = std::make_pair(b.agent_name, b.worker_id);
  {
    std::lock_guard<std::mutex> lk(m->mu);
    if (m->loaded_remotes.count(key))
      return fail(KVBM_ERR, "Remote worker already loaded: " + b.agent_name + " (worker_id=" + std::to_string(b.worker_id) + ")");
  }
  *n_out = b.layouts.size();
  if (!out) return KVBM_OK;  // size query
  if (cap < b.layouts.size()) return fail(KVBM_ERR, "handle array too small");
  // transport records
  const std::vector<uint8_t>& t = b.nixl_metadata;
  if (t.size() < 12 || std::memcmp(t.data(), kTransportMagic, 8) != 0)
    return fail(KVBM_ERR_UNSUPPORTED, "failed to load remote NIXL metadata: the blob carries no KVBM IPC transport records (a NIXL agent's "
                                      "metadata cannot be used by this library)");
  uint32_t count;
  std::memcpy(&count, t.data() + 8, 4);
  if (count != b.layouts.size()) return fail(KVBM_ERR, "transport record count does not match the layout count");
  size_t off = 12;
  std::vector<kvbm_layout_handle> done;
  auto rollback = [&](int rc) {
    const std::string msg = kvbm_last_error();
    for (kvbm_layout_handle h : done) kvbm_manager_unregister(m, h);
    return fail(rc, msg);
  };
  for (size_t i = 0; i < b.layouts.size(); ++i) {
    const kvbm_wire::Descriptor& d = b.layouts[i].layout;
    int rc = check_descriptor(d);
    if (rc) return rollback(rc);
    uint32_t blen;
    if (t.size() - off < 4) return rollback(fail(KVBM_ERR, "transport records truncated"));
    std::memcpy(&blen, t.data() + off, 4);
    off += 4;
    if (t.size() - off < blen) return rollback(fail(KVBM_ERR, "transport records truncated"));
    kvbm_layout_handle h = 0;
    rc = kvbm_manager_import_metadata(m, t.data() + off, blen, &h);
    off += blen;
    if (rc) return rollback(rc);
    done.push_back(h);
    // the descriptor and its transport record must describe the same layout
    bool same;
    {
      std::lock_guard<std::mutex> lk(m->mu);
      const Layout* L = m->find(h);
      const kvbm_layout_config c = config_of(d);
      same = L && L->cfg.num_blocks == c.num_blocks && L->cfg.num_layers == c.num_layers && L->cfg.outer_dim == c.outer_dim &&
             L->cfg.page_size == c.page_size && L->cfg.inner_dim == c.inner_dim && L->cfg.dtype_width_bytes == c.dtype_width_bytes &&
             L->fully_contiguous == d.fully_contiguous && L->allocs.size() == d.regions.size() &&
             (d.fully_contiguous || (L->block_dim == KVBM_BLOCK_IS_SECOND_DIM) == (d.block_dim == 1));
    }
    if (!same) return rollback(fail(KVBM_ERR_INCOMPATIBLE, "failed to reconstruct layout: descriptor and transport record disagree"));
  }
  for (size_t i = 0; i < done.size(); ++i) out[i] = done[i];
  std::lock_guard<std::mutex> lk(m->mu);
  m->loaded_remotes.insert(key);
  return KVBM_OK;
  });
}
