// vectorized_copy.fatbin -- drop-in for the v1 block manager's embedded kernel module.
//
// Dynamo's v1 KVBM does not link libkvbm_kernels; it cuModuleLoadData()s a fatbin and looks up the symbol
// `vectorised_copy(void** src, void** dst, size_t size, int num_pairs)`, launching it with
// grid = min(1024, num_pairs), block = 256, 0 bytes of dynamic shared memory
// (/root/reference/lib/llm/src/block_manager/block/transfer/cuda.rs:85-153, :521-548); the module can be
// replaced at run time through DYN_FATBIN_PATH (cuda.rs:588-611).  This file builds that module for sm_90a.
// The fixed launch configuration gives no workspace for a tile scheduler, so the kernel is the SIMT engine of the
// library's K1 (8 independent 16-byte loads in flight per thread, the reference's alignment ladder), pairs strided
// over the grid; pairs larger than 32 KiB are additionally split over the warps' CTAs chunk by chunk.
#include "copy_engine.cuh"

extern "C" __global__ void __launch_bounds__(256)
vectorised_copy(void** src, void** dst, size_t size, int num_pairs)
{
  using namespace kvbm;
  if (size == 0 || num_pairs <= 0) return;
  constexpr size_t kChunk = 32768;
  const size_t chunks = (size + kChunk - 1) / kChunk;
  const unsigned long long total = static_cast<unsigned long long>(num_pairs) * chunks;
  for (unsigned long long w = blockIdx.x; w < total; w += gridDim.x) {
    const unsigned long long pair = w / chunks;
    const size_t off = static_cast<size_t>(w - pair * chunks) * kChunk;
    const size_t left = size - off;
    group_copy_simt(static_cast<uint8_t*>(dst[pair]) + off, static_cast<const uint8_t*>(src[pair]) + off, left < kChunk ? left : kChunk,
                    threadIdx.x, blockDim.x);
  }
}
