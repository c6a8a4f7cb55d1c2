"""kvbench -- the reference's own KV transfer benchmark (lib/kvbm-kernels/examples/kvbench.rs), re-run on
this box against BOTH libraries through the identical C ABI:

    impl=ours       dynamo_b200/libkvbm_kernels.so            (sm_90a TMA ring)
    impl=reference  oracle/_ref/libkvbm_kernels_ref.so         (tensor_kernels.cu compiled unmodified for sm_90)

Same model (Llama 3.1 70B bf16: 80 layers, 8 KV heads, head_dim 128, K+V), same patterns (fc_to_fc: one copy
per block; lw_to_fc: one copy per (block, layer, outer)), same backends (vectorized = K1 with device pointer
tables, batched = K4 cudaMemcpyBatchAsync), same protocol (10 warm-up + 100 timed, CUDA events, median,
GB/s = total bytes / median) -- kvbench.rs:466-571.  CSV on stdout, README.md:100-156 is the published run.

    python benchmarks/kvbench.py --num-blocks 1,128 --tokens-per-block 16,64 --direction h2d,d2d --out gpurun_out/kvbench.csv
"""
import argparse
import ctypes as C
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from dynamo_b200 import kernels as K  # noqa: E402

NUM_LAYERS, NUM_KV_HEADS, HEAD_DIM, ELEM, OUTER = 80, 8, 128, 2, 2


def load_ref():
    p = os.path.join(ROOT, "oracle", "_ref", "libkvbm_kernels_ref.so")
    if not os.path.exists(p):
        return None
    L = C.CDLL(p)
    L.kvbm_kernels_launch_vectorized_copy.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_int, C.c_void_p]
    L.kvbm_kernels_memcpy_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_int, C.c_void_p]
    return L


def alloc(kind, nbytes):
    if kind == "device":
        return torch.full((nbytes,), 0xAB, dtype=torch.uint8, device="cuda")
    t = torch.empty(nbytes, dtype=torch.uint8).pin_memory()
    t.fill_(0xAB)
    return t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--num-blocks", default="1,128")
    ap.add_argument("--tokens-per-block", default="16,64")
    ap.add_argument("--backend", default="vectorized,batched")
    ap.add_argument("--direction", default="h2d,d2h,d2d")
    ap.add_argument("--pattern", default="fc_to_fc,lw_to_fc")
    ap.add_argument("--impl", default="ours,reference")
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    torch.cuda.set_device(0)
    libs = {"ours": K.lib(), "reference": load_ref()}
    stream = torch.cuda.Stream()
    sp = int(stream.cuda_stream)
    rows = ["impl,tokens_per_block,num_blocks,pattern,direction,backend,total_bytes,inner_bytes,copy_size,num_copies,median_ms,bandwidth_gbps"]
    print(rows[0], flush=True)
    for tpb in map(int, a.tokens_per_block.split(",")):
        inner = tpb * NUM_KV_HEADS * HEAD_DIM * ELEM
        block = inner * OUTER * NUM_LAYERS
        for nb in map(int, a.num_blocks.split(",")):
            total = block * nb
            for direction in a.direction.split(","):
                skind = "pinned" if direction == "h2d" else "device"
                dkind = "pinned" if direction == "d2h" else "device"
                for pattern in a.pattern.split(","):
                    dst = alloc(dkind, total)                      # FC destination [nb][layer][outer][inner]
                    if pattern == "fc_to_fc":
                        src = [alloc(skind, total)]
                        copy_size, ncopies = block, nb
                        sptr = [src[0].data_ptr() + b * block for b in range(nb)]
                        dptr = [dst.data_ptr() + b * block for b in range(nb)]
                    else:                                          # LW source: per layer [outer][nb][inner]
                        src = [alloc(skind, OUTER * nb * inner) for _ in range(NUM_LAYERS)]
                        copy_size, ncopies = inner, nb * NUM_LAYERS * OUTER
                        sptr, dptr = [], []
                        for b in range(nb):
                            for l in range(NUM_LAYERS):
                                for o in range(OUTER):
                                    sptr.append(src[l].data_ptr() + (o * nb + b) * inner)
                                    dptr.append(dst.data_ptr() + ((b * NUM_LAYERS + l) * OUTER + o) * inner)
                    st = torch.tensor(sptr, dtype=torch.int64, device="cuda")
                    dt = torch.tensor(dptr, dtype=torch.int64, device="cuda")
                    hs = (C.c_void_p * ncopies)(*sptr)
                    hd = (C.c_void_p * ncopies)(*dptr)
                    for backend in a.backend.split(","):
                        for impl in a.impl.split(","):
                            L = libs.get(impl)
                            if L is None:
                                continue
                            if backend == "vectorized":
                                fn = lambda: L.kvbm_kernels_launch_vectorized_copy(st.data_ptr(), dt.data_ptr(), copy_size, ncopies, sp)
                            else:
                                fn = lambda: L.kvbm_kernels_memcpy_batch(hs, hd, copy_size, ncopies, 0, sp)
                            iters = a.iters if total < (1 << 30) or direction == "d2d" else max(10, a.iters // 5)
                            for _ in range(a.warmup):
                                assert fn() == 0
                            stream.synchronize()
                            ts = []
                            for _ in range(iters):
                                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                                e0.record(stream)
                                assert fn() == 0
                                e1.record(stream)
                                e1.synchronize()
                                ts.append(e0.elapsed_time(e1))
                            med = statistics.median(ts)
                            rows.append(f"{impl},{tpb},{nb},{pattern},{direction},{backend},{total},{inner},{copy_size},{ncopies},{med:.4f},{total / med / 1e6:.2f}")
                            print(rows[-1], flush=True)
                    del src, dst, st, dt
                    torch.cuda.empty_cache()
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        open(a.out, "w").write("\n".join(rows) + "\n")


if __name__ == "__main__":
    main()
