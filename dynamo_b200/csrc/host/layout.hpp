// Host-side layouts: C++ restatement of lib/kvbm-physical/src/layout/{config,fully_contiguous,layer_separate}.rs
#pragma once
#include <cstddef>
#include <cstdint>
#include <exception>
#include <string>
#include <vector>

#include "../../../include/kvbm_physical.h"

namespace kvbm_host {

struct Error {
  int code;
  std::string msg;
};

inline bool is_pow2(size_t x) { return x != 0 && (x & (x - 1)) == 0; }

// layout/config.rs:16-44 (validator ranges) + :165-180 (custom validators)
inline int validate_config(const kvbm_layout_config& c, std::string* why)
{
  auto fail = [&](const char* m) {
    if (why) *why = m;
    return KVBM_ERR_CONFIG;
  };
  if (c.num_blocks < 1) return fail("num_blocks must be >= 1");
  if (c.num_layers < 1) return fail("num_layers must be >= 1");
  if (c.outer_dim < 1 || c.outer_dim > 2) return fail("outer_dim must be in 1..=2");
  if (c.page_size < 1) return fail("page_size must be >= 1");
  if (c.inner_dim < 1) return fail("inner_dim must be >= 1");
  const size_t align = c.alignment == 0 ? 1 : c.alignment;
  if (!is_pow2(align)) return fail("alignment_must_be_power_of_2");
  const size_t w = c.dtype_width_bytes;
  const bool ok = is_pow2(w) && ((w >= 2 && w <= 8) || (c.allow_fp8 && w == 1));
  if (!ok) return fail("dtype_width_bytes_must_be_power_of_two_and_less_than_8_bytes");
  return KVBM_OK;
}

// The reference multiplies with saturating_mul (config.rs:64-82): a config whose sizes do not fit a usize can never be backed
// by memory.  Configs also arrive inside metadata blobs from other processes, so every product here is overflow-checked.
inline size_t sat_mul(size_t a, size_t b)
{
  size_t r;
  return __builtin_mul_overflow(a, b, &r) ? static_cast<size_t>(-1) : r;
}
inline size_t region_size(const kvbm_layout_config& c) { return sat_mul(sat_mul(c.page_size, c.inner_dim), c.dtype_width_bytes); }
inline size_t bytes_per_block(const kvbm_layout_config& c) { return sat_mul(sat_mul(c.num_layers, c.outer_dim), region_size(c)); }
inline size_t required_bytes(const kvbm_layout_config& c) { return sat_mul(c.num_blocks, bytes_per_block(c)); }
// a layout whose total size saturates cannot exist; neither can one with more layers than bytes
inline int check_sizes(const kvbm_layout_config& c, std::string* why)
{
  if (required_bytes(c) == static_cast<size_t>(-1) || c.num_layers > (static_cast<size_t>(1) << 24)) {
    if (why) *why = "layout dimensions overflow: num_blocks * num_layers * outer_dim * page_size * inner_dim * dtype_width_bytes does not fit";
    return KVBM_ERR_CONFIG;
  }
  return KVBM_OK;
}

struct Allocation {
  uintptr_t addr;
  size_t size;
};

// One registered layout (PhysicalLayout = Layout + StorageKind + location).
struct Layout {
  kvbm_layout_config cfg{};
  bool fully_contiguous = false;
  int block_dim = KVBM_BLOCK_IS_FIRST_DIM;  // layer-separate only
  int storage = KVBM_STORAGE_SYSTEM;
  int device_id = 0;     // where the memory lives (Device storage)
  bool remote = false;   // imported from another process (peer-mapped)
  bool unmapped = false; // remote AND without a mapping in this process: descriptor only, no transfer may touch it
  int kv_block_layout = KVBM_KV_UNKNOWN;  // KvBlockLayout of one block (kv_block_layout.rs:40-76); Unknown = builder default
  size_t region = 0, block_stride = 0, layer_stride = 0, outer_stride = 0;
  std::vector<Allocation> allocs;        // 1 (FC) or num_layers (LW)
  std::vector<uint64_t> layer_base;      // address of (block 0, layer l, outer 0)
  uint64_t* dev_layer_base = nullptr;    // copy on the manager's device (kernel descriptor)

  // fully_contiguous.rs:225-257 / layer_separate.rs:215-247
  int memory_region(size_t b, size_t l, size_t o, uintptr_t* addr, size_t* size, std::string* why) const
  {
    if (b >= cfg.num_blocks) {
      if (why) *why = "Block ID " + std::to_string(b) + " out of range (count: " + std::to_string(cfg.num_blocks) + ")";
      return KVBM_ERR_RANGE;
    }
    if (l >= cfg.num_layers) {
      if (why) *why = "Layer ID " + std::to_string(l) + " out of range (count: " + std::to_string(cfg.num_layers) + ")";
      return KVBM_ERR_RANGE;
    }
    if (o >= cfg.outer_dim) {
      if (why) *why = "Outer ID " + std::to_string(o) + " out of range (count: " + std::to_string(cfg.outer_dim) + ")";
      return KVBM_ERR_RANGE;
    }
    *addr = static_cast<uintptr_t>(layer_base[l]) + b * block_stride + o * outer_stride;
    if (size) *size = region;
    return KVBM_OK;
  }
};

// FullyContiguousLayout::new_internal (fully_contiguous.rs:141-185)
inline int make_fully_contiguous(const kvbm_layout_config& cfg, uintptr_t base, size_t size, Layout* out, std::string* why)
{
  int rc = validate_config(cfg, why);
  if (rc) return rc;
  if ((rc = check_sizes(cfg, why))) return rc;
  Layout L;
  L.cfg = cfg;
  L.fully_contiguous = true;
  L.region = region_size(cfg);
  L.outer_stride = L.region;
  L.layer_stride = L.outer_stride * cfg.outer_dim;
  L.block_stride = L.layer_stride * cfg.num_layers;
  const size_t need = L.block_stride * cfg.num_blocks;
  if (size < need) {
    if (why) *why = "Memory region too small for layout. Required: " + std::to_string(need) + " bytes, got: " + std::to_string(size) + " bytes";
    return KVBM_ERR_CONFIG;
  }
  L.allocs.push_back({base, size});
  L.layer_base.resize(cfg.num_layers);
  for (size_t l = 0; l < cfg.num_layers; ++l) L.layer_base[l] = base + l * L.layer_stride;
  *out = std::move(L);
  return KVBM_OK;
}

// LayerSeparateLayout::new_internal (layer_separate.rs:155-210)
inline int make_layer_separate(const kvbm_layout_config& cfg, const uintptr_t* bases, const size_t* sizes, size_t count,
                               int block_dim, Layout* out, std::string* why)
{
  int rc = validate_config(cfg, why);
  if (rc) return rc;
  if ((rc = check_sizes(cfg, why))) return rc;
  if (count != cfg.num_layers) {
    if (why) *why = "Memory region count (" + std::to_string(count) + ") must match num_layers (" + std::to_string(cfg.num_layers) + ")";
    return KVBM_ERR_CONFIG;
  }
  if (block_dim != KVBM_BLOCK_IS_FIRST_DIM && block_dim != KVBM_BLOCK_IS_SECOND_DIM) {
    if (why) *why = "block_dim is required";
    return KVBM_ERR_CONFIG;
  }
  Layout L;
  L.cfg = cfg;
  L.fully_contiguous = false;
  L.block_dim = block_dim;
  L.region = region_size(cfg);
  if (block_dim == KVBM_BLOCK_IS_SECOND_DIM) {
    L.block_stride = L.region;
    L.outer_stride = L.block_stride * cfg.num_blocks;
  } else {
    L.outer_stride = L.region;
    L.block_stride = L.outer_stride * cfg.outer_dim;
  }
  const size_t need = cfg.num_blocks * cfg.outer_dim * L.region;
  for (size_t i = 0; i < count; ++i) {
    if (sizes[i] < need) {
      if (why) *why = "Memory region " + std::to_string(i) + " too small for layout. Required: " + std::to_string(need) + " bytes, got: " + std::to_string(sizes[i]) + " bytes";
      return KVBM_ERR_CONFIG;
    }
    L.allocs.push_back({bases[i], sizes[i]});
    L.layer_base.push_back(bases[i]);
  }
  *out = std::move(L);
  return KVBM_OK;
}

// records the thread's last error message (kvbm_last_error) and returns `code`; defined in transfer_manager.cpp
int set_last_error(int code, const std::string& msg);

// Runs the body of a C ABI entry point: no exception may cross the C boundary, so one that escapes `body` becomes KVBM_ERR with
// an "internal error" message.
template <class F>
int guarded(F&& body)
{
  try {
    return body();
  } catch (const std::exception& e) {
    return set_last_error(KVBM_ERR, std::string("internal error: ") + e.what());
  } catch (...) {
    return set_last_error(KVBM_ERR, "internal error");
  }
}

}  // namespace kvbm_host
