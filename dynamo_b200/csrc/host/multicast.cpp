// NVLS multicast groups: the 1 -> N replicate of the KV hand-off done by the NVSwitch.
//
// The reference broadcasts identical KV blocks with one ncclBcast per region inside a group
// (lib/kvbm-engine/src/collectives/nccl.rs:421-462; v1 lib/llm/src/block_manager/distributed/transfer.rs:396-475).
// Here the receivers' pools are physical allocations bound to ONE CUmulticastObject; the source GPU maps the object
// and the transfer kernel writes every tile once to the multicast address (kvbm_paged_copy_opts.multicast): NVLink
// egress of the source is 1x the payload instead of Nx, and the receivers run nothing.
//
// Only the CUDA driver's virtual-memory-management / multicast API is used, resolved through
// cudaGetDriverEntryPoint so that the library still loads (and says so loudly) where libcuda is absent.
#include <cuda.h>
#include <cuda_runtime_api.h>
#include <unistd.h>

#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "layout.hpp"

namespace {

using kvbm_host::set_last_error;

struct Driver {
  CUresult (*MulticastCreate)(CUmemGenericAllocationHandle*, const CUmulticastObjectProp*);
  CUresult (*MulticastAddDevice)(CUmemGenericAllocationHandle, CUdevice);
  CUresult (*MulticastBindMem)(CUmemGenericAllocationHandle, size_t, CUmemGenericAllocationHandle, size_t, size_t, unsigned long long);
  CUresult (*MulticastBindAddr)(CUmemGenericAllocationHandle, size_t, CUdeviceptr, size_t, unsigned long long);
  CUresult (*MulticastUnbind)(CUmemGenericAllocationHandle, CUdevice, size_t, size_t);
  CUresult (*MulticastGetGranularity)(size_t*, const CUmulticastObjectProp*, CUmulticastGranularity_flags);
  CUresult (*MemCreate)(CUmemGenericAllocationHandle*, size_t, const CUmemAllocationProp*, unsigned long long);
  CUresult (*MemRelease)(CUmemGenericAllocationHandle);
  CUresult (*MemAddressReserve)(CUdeviceptr*, size_t, size_t, CUdeviceptr, unsigned long long);
  CUresult (*MemAddressFree)(CUdeviceptr, size_t);
  CUresult (*MemMap)(CUdeviceptr, size_t, size_t, CUmemGenericAllocationHandle, unsigned long long);
  CUresult (*MemUnmap)(CUdeviceptr, size_t);
  CUresult (*MemSetAccess)(CUdeviceptr, size_t, const CUmemAccessDesc*, size_t);
  CUresult (*MemExportToShareableHandle)(void*, CUmemGenericAllocationHandle, CUmemAllocationHandleType, unsigned long long);
  CUresult (*MemImportFromShareableHandle)(CUmemGenericAllocationHandle*, void*, CUmemAllocationHandleType);
  CUresult (*MemGetAllocationGranularity)(size_t*, const CUmemAllocationProp*, CUmemAllocationGranularity_flags);
  CUresult (*DeviceGet)(CUdevice*, int);
  CUresult (*DeviceGetAttribute)(int*, CUdevice_attribute, CUdevice);
  bool ok = false;
  std::string why;
};

template <class F>
bool resolve(const char* name, F* out, std::string* why)
{
  void* f = nullptr;
  cudaDriverEntryPointQueryResult q;
  cudaError_t e = cudaGetDriverEntryPoint(name, &f, cudaEnableDefault, &q);
  if (e != cudaSuccess || f == nullptr) {
    (void)cudaGetLastError();
    *why = std::string("CUDA driver entry point ") + name + " unavailable (" + cudaGetErrorName(e) + ")";
    return false;
  }
  *out = reinterpret_cast<F>(f);
  return true;
}

Driver& driver()
{
  static Driver d = [] {
    Driver x{};
    x.ok = resolve("cuMulticastCreate", &x.MulticastCreate, &x.why) && resolve("cuMulticastAddDevice", &x.MulticastAddDevice, &x.why) &&
           resolve("cuMulticastBindMem", &x.MulticastBindMem, &x.why) && resolve("cuMulticastBindAddr", &x.MulticastBindAddr, &x.why) && resolve("cuMulticastUnbind", &x.MulticastUnbind, &x.why) &&
           resolve("cuMulticastGetGranularity", &x.MulticastGetGranularity, &x.why) && resolve("cuMemCreate", &x.MemCreate, &x.why) &&
           resolve("cuMemRelease", &x.MemRelease, &x.why) && resolve("cuMemAddressReserve", &x.MemAddressReserve, &x.why) &&
           resolve("cuMemAddressFree", &x.MemAddressFree, &x.why) && resolve("cuMemMap", &x.MemMap, &x.why) &&
           resolve("cuMemUnmap", &x.MemUnmap, &x.why) && resolve("cuMemSetAccess", &x.MemSetAccess, &x.why) &&
           resolve("cuMemExportToShareableHandle", &x.MemExportToShareableHandle, &x.why) &&
           resolve("cuMemImportFromShareableHandle", &x.MemImportFromShareableHandle, &x.why) &&
           resolve("cuMemGetAllocationGranularity", &x.MemGetAllocationGranularity, &x.why) &&
           resolve("cuDeviceGet", &x.DeviceGet, &x.why) && resolve("cuDeviceGetAttribute", &x.DeviceGetAttribute, &x.why);
    return x;
  }();
  return d;
}

int fail_cu(CUresult r, const char* what)
{
  return set_last_error(KVBM_ERR_CUDA, std::string(what) + " failed: CUresult " + std::to_string(static_cast<int>(r)));
}
#define DRV(call)                                   \
  do {                                              \
    CUresult r__ = (call);                          \
    if (r__ != CUDA_SUCCESS) return fail_cu(r__, #call); \
  } while (0)

// make sure the device's primary context exists (the VMM calls need an initialised device)
int touch_device(int device)
{
  int prev = -1;
  cudaError_t e = cudaGetDevice(&prev);
  if (e == cudaSuccess) e = cudaSetDevice(device);
  if (e == cudaSuccess) e = cudaFree(nullptr);
  if (prev >= 0) (void)cudaSetDevice(prev);
  if (e != cudaSuccess) {
    (void)cudaGetLastError();
    return set_last_error(KVBM_ERR_CUDA, std::string("cannot initialise CUDA device ") + std::to_string(device) + ": " + cudaGetErrorName(e));
  }
  return KVBM_OK;
}

struct Member {
  int device = -1;
  CUmemGenericAllocationHandle mem = 0;
  CUdeviceptr va = 0;
  bool bound = false;
  bool owned = true;   // false: the engine's own allocation bound with cuMulticastBindAddr -- never unmapped / released here
};
struct Mapping {
  int device = -1;
  CUdeviceptr va = 0;
};

}  // namespace

struct kvbm_mc_group {
  CUmemGenericAllocationHandle mc = 0;
  int num_devices = 0;
  size_t size = 0;        // bytes bound per device (rounded)
  size_t va_align = 0;
  bool shareable = false;
  std::vector<Member> members;    // devices THIS process bound memory for
  std::vector<Mapping> mappings;  // multicast mappings THIS process created
};

namespace {

CUmulticastObjectProp mc_prop(int num_devices, size_t size, bool shareable)
{
  CUmulticastObjectProp p;
  std::memset(&p, 0, sizeof p);
  p.numDevices = static_cast<unsigned>(num_devices);
  p.size = size;
  p.handleTypes = shareable ? CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR : 0;
  return p;
}

// bound size: a multiple of the multicast granularity -- the RECOMMENDED one (queried from the driver) for pools that are
// at least that large, the MINIMUM (2 MiB) for small ones
int round_size(int num_devices, size_t bytes, bool shareable, size_t* rounded, size_t* va_align)
{
  Driver& d = driver();
  CUmulticastObjectProp p = mc_prop(num_devices, bytes, shareable);
  size_t gmin = 0, grec = 0;
  DRV(d.MulticastGetGranularity(&gmin, &p, CU_MULTICAST_GRANULARITY_MINIMUM));
  DRV(d.MulticastGetGranularity(&grec, &p, CU_MULTICAST_GRANULARITY_RECOMMENDED));
  if (gmin == 0) gmin = 2u << 20;
  if (grec < gmin) grec = gmin;
  const size_t g = bytes >= grec ? grec : gmin;
  *rounded = (bytes + g - 1) / g * g;
  *va_align = grec;
  return KVBM_OK;
}

int check_ready(const kvbm_mc_group* g)
{
  if (!g) return set_last_error(KVBM_ERR_HANDLE, "null multicast group");
  Driver& d = driver();
  if (!d.ok) return set_last_error(KVBM_ERR_CUDA, d.why);
  return KVBM_OK;
}

}  // namespace

extern "C" int kvbm_mc_supported(int device)
{
  Driver& d = driver();
  if (!d.ok) {
    set_last_error(KVBM_ERR_CUDA, d.why);
    return 0;
  }
  if (touch_device(device) != KVBM_OK) return 0;
  CUdevice dev;
  int v = 0;
  if (d.DeviceGet(&dev, device) != CUDA_SUCCESS) return 0;
  if (d.DeviceGetAttribute(&v, CU_DEVICE_ATTRIBUTE_MULTICAST_SUPPORTED, dev) != CUDA_SUCCESS) return 0;
  return v != 0;
}

extern "C" int kvbm_mc_group_create(int num_devices, size_t bytes_per_device, int shareable, kvbm_mc_group** out)
{
  try {
  if (!out || num_devices < 1 || bytes_per_device == 0) return set_last_error(KVBM_ERR, "bad multicast group arguments");
  Driver& d = driver();
  if (!d.ok) return set_last_error(KVBM_ERR_CUDA, d.why);
  int dev0 = 0;
  (void)cudaGetDevice(&dev0);
  int rc = touch_device(dev0);
  if (rc) return rc;
  auto g = new kvbm_mc_group();
  g->num_devices = num_devices;
  g->shareable = shareable != 0;
  rc = round_size(num_devices, bytes_per_device, g->shareable, &g->size, &g->va_align);
  if (rc) {
    delete g;
    return rc;
  }
  CUmulticastObjectProp p = mc_prop(num_devices, g->size, g->shareable);
  CUresult r = d.MulticastCreate(&g->mc, &p);
  if (r != CUDA_SUCCESS) {
    delete g;
    return fail_cu(r, "cuMulticastCreate");
  }
  *out = g;
  return KVBM_OK;
  } catch (const std::exception& e) {
    return kvbm_host::set_last_error(KVBM_ERR, std::string("internal error: ") + e.what());
  } catch (...) {
    return kvbm_host::set_last_error(KVBM_ERR, "internal error");
  }
}

extern "C" int kvbm_mc_group_export_fd(kvbm_mc_group* g, int* fd)
{
  try {
  int rc = check_ready(g);
  if (rc) return rc;
  if (!fd) return set_last_error(KVBM_ERR, "null fd");
  if (!g->shareable) return set_last_error(KVBM_ERR, "multicast group was not created shareable");
  int h = -1;
  DRV(driver().MemExportToShareableHandle(&h, g->mc, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR, 0));
  *fd = h;
  return KVBM_OK;
  } catch (const std::exception& e) {
    return kvbm_host::set_last_error(KVBM_ERR, std::string("internal error: ") + e.what());
  } catch (...) {
    return kvbm_host::set_last_error(KVBM_ERR, "internal error");
  }
}

extern "C" int kvbm_mc_group_import_fd(int fd, int num_devices, size_t bytes_per_device, kvbm_mc_group** out)
{
  try {
  if (!out || fd < 0 || num_devices < 1 || bytes_per_device == 0) return set_last_error(KVBM_ERR, "bad multicast import arguments");
  Driver& d = driver();
  if (!d.ok) return set_last_error(KVBM_ERR_CUDA, d.why);
  int dev0 = 0;
  (void)cudaGetDevice(&dev0);
  int rc = touch_device(dev0);
  if (rc) return rc;
  auto g = new kvbm_mc_group();
  g->num_devices = num_devices;
  g->shareable = true;
  rc = round_size(num_devices, bytes_per_device, true, &g->size, &g->va_align);
  if (rc) {
    delete g;
    return rc;
  }
  CUresult r = d.MemImportFromShareableHandle(&g->mc, reinterpret_cast<void*>(static_cast<uintptr_t>(fd)), CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR);
  if (r != CUDA_SUCCESS) {
    delete g;
    return fail_cu(r, "cuMemImportFromShareableHandle");
  }
  *out = g;
  return KVBM_OK;
  } catch (const std::exception& e) {
    return kvbm_host::set_last_error(KVBM_ERR, std::string("internal error: ") + e.what());
  } catch (...) {
    return kvbm_host::set_last_error(KVBM_ERR, "internal error");
  }
}

extern "C" size_t kvbm_mc_group_size(const kvbm_mc_group* g) { return g ? g->size : 0; }

extern "C" int kvbm_mc_group_add_device(kvbm_mc_group* g, int device)
{
  try {
  int rc = check_ready(g);
  if (rc) return rc;
  if ((rc = touch_device(device))) return rc;
  CUdevice dev;
  DRV(driver().DeviceGet(&dev, device));
  DRV(driver().MulticastAddDevice(g->mc, dev));
  return KVBM_OK;
  } catch (const std::exception& e) {
    return kvbm_host::set_last_error(KVBM_ERR, std::string("internal error: ") + e.what());
  } catch (...) {
    return kvbm_host::set_last_error(KVBM_ERR, "internal error");
  }
}

extern "C" int kvbm_mc_group_bind_local(kvbm_mc_group* g, int device, void** unicast_ptr)
{
  try {
  int rc = check_ready(g);
  if (rc) return rc;
  if (!unicast_ptr) return set_last_error(KVBM_ERR, "null out pointer");
  if ((rc = touch_device(device))) return rc;
  Driver& d = driver();
  CUmemAllocationProp ap;
  std::memset(&ap, 0, sizeof ap);
  ap.type = CU_MEM_ALLOCATION_TYPE_PINNED;
  ap.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
  ap.location.id = device;
  ap.requestedHandleTypes = g->shareable ? CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR : CU_MEM_HANDLE_TYPE_NONE;
  Member mb;
  mb.device = device;
  DRV(d.MemCreate(&mb.mem, g->size, &ap, 0));
  CUresult r = d.MemAddressReserve(&mb.va, g->size, g->va_align, 0, 0);
  if (r == CUDA_SUCCESS) r = d.MemMap(mb.va, g->size, 0, mb.mem, 0);
  if (r == CUDA_SUCCESS) {
    // the owner and every peer this process can reach over P2P: the pool stays usable for ordinary (unicast)
    // transfers next to the multicast ones
    std::vector<CUmemAccessDesc> ads;
    int count = 0;
    (void)cudaGetDeviceCount(&count);
    for (int p = 0; p < count; ++p) {
      int can = p == device;
      if (!can && cudaDeviceCanAccessPeer(&can, p, device) != cudaSuccess) {
        (void)cudaGetLastError();
        can = 0;
      }
      if (!can) continue;
      CUmemAccessDesc ad;
      std::memset(&ad, 0, sizeof ad);
      ad.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
      ad.location.id = p;
      ad.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
      ads.push_back(ad);
    }
    r = d.MemSetAccess(mb.va, g->size, ads.data(), ads.size());
  }
  if (r == CUDA_SUCCESS) r = d.MulticastBindMem(g->mc, 0, mb.mem, 0, g->size, 0);
  if (r != CUDA_SUCCESS) {
    if (mb.va) {
      d.MemUnmap(mb.va, g->size);
      d.MemAddressFree(mb.va, g->size);
    }
    d.MemRelease(mb.mem);
    return fail_cu(r, "multicast bind (cuMemAddressReserve / cuMemMap / cuMemSetAccess / cuMulticastBindMem)");
  }
  mb.bound = true;
  g->members.push_back(mb);
  *unicast_ptr = reinterpret_cast<void*>(mb.va);
  return KVBM_OK;
  } catch (const std::exception& e) {
    return kvbm_host::set_last_error(KVBM_ERR, std::string("internal error: ") + e.what());
  } catch (...) {
    return kvbm_host::set_last_error(KVBM_ERR, "internal error");
  }
}

// Bind memory the ENGINE already owns (a KV pool it allocated itself) instead of allocating a pool here: the range must be
// backed by the driver's virtual-memory-management API (cuMemCreate + cuMemMap -- e.g. PyTorch's expandable segments) and
// aligned to the multicast granularity.  The first kvbm_mc_group_size() bytes of `ptr` become this device's share.
extern "C" int kvbm_mc_group_bind_addr(kvbm_mc_group* g, int device, void* ptr, size_t bytes)
{
  try {
  int rc = check_ready(g);
  if (rc) return rc;
  if (!ptr || bytes < g->size) return set_last_error(KVBM_ERR, "bind_addr: the range must cover kvbm_mc_group_size() bytes");
  if ((rc = touch_device(device))) return rc;
  CUresult r = driver().MulticastBindAddr(g->mc, 0, reinterpret_cast<CUdeviceptr>(ptr), g->size, 0);
  if (r != CUDA_SUCCESS)
    return fail_cu(r, "cuMulticastBindAddr (is the range cuMemCreate-backed and granularity-aligned?)");
  Member mb;
  mb.device = device;
  mb.va = reinterpret_cast<CUdeviceptr>(ptr);
  mb.bound = true;
  mb.owned = false;
  g->members.push_back(mb);
  return KVBM_OK;
  } catch (const std::exception& e) {
    return kvbm_host::set_last_error(KVBM_ERR, std::string("internal error: ") + e.what());
  } catch (...) {
    return kvbm_host::set_last_error(KVBM_ERR, "internal error");
  }
}

extern "C" int kvbm_mc_group_map(kvbm_mc_group* g, int device, void** multicast_ptr)
{
  try {
  int rc = check_ready(g);
  if (rc) return rc;
  if (!multicast_ptr) return set_last_error(KVBM_ERR, "null out pointer");
  if ((rc = touch_device(device))) return rc;
  Driver& d = driver();
  Mapping mp;
  mp.device = device;
  DRV(d.MemAddressReserve(&mp.va, g->size, g->va_align, 0, 0));
  CUresult r = d.MemMap(mp.va, g->size, 0, g->mc, 0);
  if (r == CUDA_SUCCESS) {
    CUmemAccessDesc ad;
    std::memset(&ad, 0, sizeof ad);
    ad.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
    ad.location.id = device;
    ad.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
    r = d.MemSetAccess(mp.va, g->size, &ad, 1);
    if (r != CUDA_SUCCESS) d.MemUnmap(mp.va, g->size);
  }
  if (r != CUDA_SUCCESS) {
    d.MemAddressFree(mp.va, g->size);
    return fail_cu(r, "multicast map (cuMemMap / cuMemSetAccess)");
  }
  g->mappings.push_back(mp);
  *multicast_ptr = reinterpret_cast<void*>(mp.va);
  return KVBM_OK;
  } catch (const std::exception& e) {
    return kvbm_host::set_last_error(KVBM_ERR, std::string("internal error: ") + e.what());
  } catch (...) {
    return kvbm_host::set_last_error(KVBM_ERR, "internal error");
  }
}

extern "C" void kvbm_mc_group_destroy(kvbm_mc_group* g)
{
  if (!g) return;
  Driver& d = driver();
  const bool trace = std::getenv("KVBM_MC_TRACE") != nullptr;
  auto now = [] { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); };
  double t0 = now();
  auto step = [&](const char* what) {
    if (!trace) return;
    const double t1 = now();
    std::fprintf(stderr, "[kvbm_mc] %s: %.3f s\n", what, t1 - t0);
    t0 = t1;
  };
  if (d.ok) {
    for (auto& mp : g->mappings) {
      d.MemUnmap(mp.va, g->size);
      d.MemAddressFree(mp.va, g->size);
    }
    step("unmap multicast ranges");
    for (auto& mb : g->members) {
      CUdevice dev;
      if (mb.bound && d.DeviceGet(&dev, mb.device) == CUDA_SUCCESS) d.MulticastUnbind(g->mc, dev, 0, g->size);
      step("unbind");
      if (!mb.owned) continue;
      d.MemUnmap(mb.va, g->size);
      d.MemAddressFree(mb.va, g->size);
      step("unmap pool");
      d.MemRelease(mb.mem);
      step("release pool");
    }
    if (g->mc) d.MemRelease(g->mc);
    step("release multicast object");
  }
  delete g;
}
