// Bench-only baseline: the reference's 1 -> N replicate, i.e. ONE ncclBcast PER (block, layer, outer) REGION inside a
// group (kvbm-engine collectives/nccl.rs:321-356 `broadcast_regions`, :366-390 `collect_regions`, :421-462 `broadcast`;
// root = rank 0 sends from its src blocks, every other rank receives into its dst blocks).  Single process, one
// communicator per visible GPU (ncclCommInitAll), vLLM layer-separate pools, Llama-3-8B geometry.
// Prints one JSON line; compare with `bench.py --replicate [--nvls]`.  Not part of the product libraries.
//
//   nvcc -O2 -std=c++17 -gencode arch=compute_90a,code=sm_90a -o benchmarks/nccl_bcast_baseline \
//        benchmarks/nccl_bcast_baseline.cu -lnccl
#include <cuda_runtime_api.h>
#include <nccl.h>

#include <algorithm>
#include <chrono>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <numeric>
#include <random>
#include <vector>

#define CK(x)                                                                            \
  do {                                                                                   \
    cudaError_t e__ = (x);                                                               \
    if (e__ != cudaSuccess) {                                                            \
      std::fprintf(stderr, "%s failed: %s\n", #x, cudaGetErrorString(e__));              \
      std::exit(2);                                                                      \
    }                                                                                    \
  } while (0)
#define NK(x)                                                                            \
  do {                                                                                   \
    ncclResult_t r__ = (x);                                                              \
    if (r__ != ncclSuccess) {                                                            \
      std::fprintf(stderr, "%s failed: %s\n", #x, ncclGetErrorString(r__));              \
      std::exit(3);                                                                      \
    }                                                                                    \
  } while (0)

int main(int argc, char** argv)
{
  int blocks = 256, pool = 1024, layers = 32, iters = 10, warmup = 2;
  for (int i = 1; i + 1 < argc; i += 2) {
    const std::string k = argv[i];
    const int v = std::atoi(argv[i + 1]);
    if (k == "--blocks") blocks = v;
    else if (k == "--pool") pool = v;
    else if (k == "--layers") layers = v;
    else if (k == "--iters") iters = v;
    else if (k == "--warmup") warmup = v;
  }
  const size_t region = 16 * 1024 * 2, outer = 2;  // page 16 x inner 1024 x bf16
  int n = 0;
  CK(cudaGetDeviceCount(&n));
  if (n < 2) {
    std::fprintf(stderr, "needs >= 2 GPUs\n");
    return 1;
  }
  std::vector<int> devs(n);
  std::iota(devs.begin(), devs.end(), 0);
  std::vector<ncclComm_t> comm(n);
  NK(ncclCommInitAll(comm.data(), n, devs.data()));
  std::vector<cudaStream_t> st(n);
  std::vector<std::vector<uint8_t*>> bufs(n, std::vector<uint8_t*>(layers));   // [rank][layer] -> [outer][pool][region]
  for (int r = 0; r < n; ++r) {
    CK(cudaSetDevice(r));
    CK(cudaStreamCreateWithFlags(&st[r], cudaStreamNonBlocking));
    for (int l = 0; l < layers; ++l) {
      CK(cudaMalloc(&bufs[r][l], outer * pool * region));
      CK(cudaMemset(bufs[r][l], r == 0 ? 0x5a + l : 0, outer * pool * region));
    }
  }
  // block tables: root uses src ids, the others dst ids (nccl.rs:432-443); random, non-contiguous
  std::vector<int> src(pool), dst(pool);
  std::iota(src.begin(), src.end(), 0);
  std::iota(dst.begin(), dst.end(), 0);
  std::shuffle(src.begin(), src.end(), std::mt19937(10));
  std::shuffle(dst.begin(), dst.end(), std::mt19937(100));
  // collect_regions order: block, layer, outer
  std::vector<std::vector<uint8_t*>> regions(n);
  for (int r = 0; r < n; ++r)
    for (int b = 0; b < blocks; ++b)
      for (int l = 0; l < layers; ++l)
        for (size_t o = 0; o < outer; ++o)
          regions[r].push_back(bufs[r][l] + (o * pool + (r == 0 ? src[b] : dst[b])) * region);
  const size_t nreg = regions[0].size();
  auto once = [&]() {
    NK(ncclGroupStart());
    for (int r = 0; r < n; ++r)
      for (size_t i = 0; i < nreg; ++i) NK(ncclBcast(regions[r][i], region, ncclChar, 0, comm[r], st[r]));
    NK(ncclGroupEnd());
    for (int r = 0; r < n; ++r) {
      CK(cudaSetDevice(r));
      CK(cudaStreamSynchronize(st[r]));
    }
  };
  for (int i = 0; i < warmup; ++i) once();
  std::vector<double> ms;
  for (int i = 0; i < iters; ++i) {
    const auto t0 = std::chrono::steady_clock::now();
    once();
    ms.push_back(std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count());
  }
  std::sort(ms.begin(), ms.end());
  const double med = ms[ms.size() / 2];
  // verify one block on the last rank
  std::vector<uint8_t> a(region), b(region);
  CK(cudaSetDevice(0));
  CK(cudaMemcpy(a.data(), regions[0][nreg - 1], region, cudaMemcpyDeviceToHost));
  CK(cudaSetDevice(n - 1));
  CK(cudaMemcpy(b.data(), regions[n - 1][nreg - 1], region, cudaMemcpyDeviceToHost));
  const bool ok = a == b;
  const double payload = static_cast<double>(nreg) * region;
  std::printf("{\"baseline\": \"ncclBcast per region, grouped (kvbm-engine nccl.rs:321-356)\", \"gpus\": %d, \"regions\": %zu, "
              "\"payload_bytes\": %.0f, \"ms_median\": %.4f, \"delivered_gbs_all_destinations\": %.2f, \"per_destination_gbs\": %.2f, "
              "\"includes\": \"host enqueue of every ncclBcast + stream sync\", \"bit_exact_probe\": %s}\n",
              n, nreg, payload, med, payload * (n - 1) / med / 1e6, payload / med / 1e6, ok ? "true" : "false");
  for (int r = 0; r < n; ++r) ncclCommDestroy(comm[r]);
  return ok ? 0 : 4;
}
