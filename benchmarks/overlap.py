"""Layer-streamed KV push overlapped with (stand-in) attention -- BASELINE configs[3] per rank pair.

Llama-3-70B TP=4 shard: 80 layers, 2 KV heads/rank -> 8 KiB regions, 256 blocks (4k ctx) = 4 MiB per layer.
Main stream: per layer an HBM-bound stand-in for attention (~--layer-us), then release layer l.
Transfer:  (ours)  ONE launch of the paged kernel on a side stream, gated per layer by ready flags, capped to
                   --ctas CTAs so the compute keeps the rest of the chip; publishes per-layer done flags.
           (ref-style) the reference's pattern (lib/kvbm-engine/src/worker/physical.rs:277-346): per layer an event
                   + one K1 launch with host-built pointer tables for that layer.
Reports T_compute, T_transfer, T_overlapped and hidden fraction = (Tc + Tt - To) / Tt.
With 2 visible GPUs the destination pool lives on GPU 1 (NVLink peer stores); otherwise same GPU.
"""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from dynamo_b200 import kernels as K  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--layers", type=int, default=80)
ap.add_argument("--inner", type=int, default=256)
ap.add_argument("--blocks", type=int, default=256)
ap.add_argument("--pool", type=int, default=2048)
ap.add_argument("--layer-us", type=float, default=40.0)
ap.add_argument("--ctas", type=int, default=16)
ap.add_argument("--iters", type=int, default=10)
ap.add_argument("--standin-blocks", type=int, default=132 * 4)
ap.add_argument("--fma", type=int, default=0, help="dependent FMA pairs per 16 B: >0 makes the stand-in compute-bound instead of HBM-saturating")
ap.add_argument("--warps", type=int, default=0)
ap.add_argument("--stages", type=int, default=0)
ap.add_argument("--tile", type=int, default=0)
ap.add_argument("--standin", choices=["stream", "gemm"], default="stream",
                help="stream: the synthetic streaming/FMA kernel; gemm: a real tensor-core layer (cuBLAS bf16 GEMM chain via torch.matmul)")
ap.add_argument("--gemm-n", type=int, default=4096)
ap.add_argument("--out", default="gpurun_out/overlap.json")
a = ap.parse_args()

torch.cuda.set_device(0)
peer = torch.cuda.device_count() > 1
ddev = "cuda:1" if peer else "cuda:0"
if peer:
    from dynamo_b200.physical import TransferManager
    _m = TransferManager(device=0)
    _m.enable_peer_access(1)
nl, nbp, n = a.layers, a.pool, a.blocks
region = 16 * a.inner * 2


def pool(dev):
    bufs = [torch.empty(2 * nbp * region, dtype=torch.uint8, device=dev) for _ in range(nl)]
    base = torch.tensor([b.data_ptr() for b in bufs], dtype=torch.int64, device="cuda:0")
    return bufs, base, K.PagedLayout(base.data_ptr(), region, region * nbp, region, nl, 2, nbp)


sb, sbase, src = pool("cuda:0")
db, dbase, dst = pool(ddev)
for t in sb:
    t.random_(0, 256)
sid = torch.from_numpy(np.random.default_rng(0).permutation(nbp)[:n].astype(np.int32)).cuda()
did = torch.from_numpy(np.random.default_rng(1).permutation(nbp)[:n].astype(np.int32)).cuda()
ready = torch.zeros(nl, dtype=torch.int32, device="cuda:0")
done = torch.zeros(nl, dtype=torch.int32, device=ddev)
ws = torch.zeros(nl + 4, dtype=torch.int32, device="cuda:0")
main = torch.cuda.current_stream()
side = torch.cuda.Stream(priority=-1)   # the persistent transfer CTAs should win SM slots as compute CTAs retire
mp, sp = int(main.cuda_stream), int(side.cuda_stream)

# stand-in attention: copy sized to take ~layer-us at ~6 TB/s r+w
work_bytes = int(a.layer_us * 1e-6 * 5.0e12 / 2) if a.fma == 0 else int(a.layer_us * 1e-6 * 5.0e12 / 2 / max(1.0, a.fma / 24.0))
wa = torch.empty(work_bytes, dtype=torch.uint8, device="cuda:0")
wb = torch.empty_like(wa)


_standin_path = os.path.join(ROOT, "benchmarks", "libstandin.so")
SL = C.CDLL(_standin_path)
SL.standin_attention_layer.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_uint32, C.c_void_p, C.c_int, C.c_int, C.c_void_p]
counter = torch.zeros(1, dtype=torch.int32, device="cuda:0")
n_vec = work_bytes // 16
standin_blocks = a.standin_blocks   # keep it well below a full wave: a grid that exactly fills the chip gets a second wave when anything else is resident


if a.standin == "gemm":
    gA = torch.randn(a.gemm_n, a.gemm_n, dtype=torch.bfloat16, device="cuda:0")
    gB = torch.randn(a.gemm_n, a.gemm_n, dtype=torch.bfloat16, device="cuda:0")
    gC = torch.empty_like(gA)


def compute_layer(flag_ptr=0, value=0):
    if a.standin == "gemm":
        # a real prefill-shaped layer: one cuBLAS bf16 GEMM (wgmma kernel on sm_90, ~1 CTA/SM, large smem); the ready flag is
        # released by a stream mem-op right behind it
        torch.matmul(gA, gB, out=gC)
        if flag_ptr:
            K.check(K.set_flags(flag_ptr, 0, 1, value, mp))
        return
    # SM kernel, HBM-bound (16 B read + 16 B written per thread-iteration): stands in for attention; when flag_ptr is
    # given its last block releases that layer's ready flag (what an engine's KV-write epilogue would do)
    assert SL.standin_attention_layer(wa.data_ptr(), wb.data_ptr(), n_vec, flag_ptr, value, counter.data_ptr(), standin_blocks, a.fma, mp) == 0


def t_ms(fn, iters):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(main)
        fn()
        e1.record(main)
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return float(np.median(ts))


epoch = [0]


def compute_only():
    for _ in range(nl):
        compute_layer()


def compute_and_signal():   # the producer-side cost of releasing layers, without any transfer
    epoch[0] += 1
    for l in range(nl):
        compute_layer(ready[l:].data_ptr(), epoch[0])


def transfer_only(ctas):
    d = K.PagedDst(dst, sid.data_ptr(), did.data_ptr(), 0, 0)
    K.check(K.paged_copy(src, [d], n, 0, nl, 0, K.PagedCopyOpts(max_ctas=ctas, warps_per_cta=a.warps, stages=a.stages, tile_bytes=a.tile), mp))


def overlapped_ours():
    epoch[0] += 1
    e = epoch[0]
    d = K.PagedDst(dst, sid.data_ptr(), did.data_ptr(), 0, done.data_ptr())
    opts = K.PagedCopyOpts(epoch=e, layer_ready_flags=ready.data_ptr(), sync_workspace=ws.data_ptr(), max_ctas=a.ctas,
                           warps_per_cta=a.warps, stages=a.stages, tile_bytes=a.tile)
    side.wait_stream(main)
    K.check(K.paged_copy(src, [d], n, 0, nl, 0, opts, sp))
    for l in range(nl):
        compute_layer(ready[l:].data_ptr(), e)
    main.wait_stream(side)


helper = torch.cuda.Stream(priority=-1)
hp = int(helper.cuda_stream)
layer_events = [torch.cuda.Event() for _ in range(nl)]


def overlapped_ours_events():
    """Integration-realistic signalling: the worker already records one event per layer
    (connector_worker.py:226); a helper stream turns each event into a ready-flag write (cuStreamWriteValue32),
    so the compute stream carries nothing extra and the transfer is still ONE launch."""
    epoch[0] += 1
    e = epoch[0]
    d = K.PagedDst(dst, sid.data_ptr(), did.data_ptr(), 0, done.data_ptr())
    opts = K.PagedCopyOpts(epoch=e, layer_ready_flags=ready.data_ptr(), sync_workspace=ws.data_ptr(), max_ctas=a.ctas,
                           warps_per_cta=a.warps, stages=a.stages, tile_bytes=a.tile)
    side.wait_stream(main)
    K.check(K.paged_copy(src, [d], n, 0, nl, 0, opts, sp))
    for l in range(nl):
        compute_layer()
        layer_events[l].record(main)
        helper.wait_event(layer_events[l])
        K.check(K.set_flags(ready.data_ptr(), l, 1, e, hp))
    main.wait_stream(side)


def overlapped_ours_per_layer():
    """The reference's pattern (physical.rs:277-346) with OUR kernel: one event + one capped launch per layer."""
    d = K.PagedDst(dst, sid.data_ptr(), did.data_ptr(), 0, 0)
    opts = K.PagedCopyOpts(max_ctas=a.ctas, warps_per_cta=a.warps, stages=a.stages, tile_bytes=a.tile)
    for l in range(nl):
        compute_layer()
        layer_events[l].record(main)
        side.wait_event(layer_events[l])
        K.check(K.paged_copy(src, [d], n, l, l + 1, 0, opts, sp))
    main.wait_stream(side)


def overlapped_ours_prereleased():
    """Diagnostic: every layer released up front -> the transfer runs ungated next to the first layers only."""
    epoch[0] += 1
    e = epoch[0]
    d = K.PagedDst(dst, sid.data_ptr(), did.data_ptr(), 0, done.data_ptr())
    opts = K.PagedCopyOpts(epoch=e, layer_ready_flags=ready.data_ptr(), sync_workspace=ws.data_ptr(), max_ctas=a.ctas,
                           warps_per_cta=a.warps, stages=a.stages, tile_bytes=a.tile)
    K.check(K.set_flags(ready.data_ptr(), 0, nl, e, mp))
    side.wait_stream(main)
    K.check(K.paged_copy(src, [d], n, 0, nl, 0, opts, sp))
    pre_ev[1].record(side)
    for l in range(nl):
        compute_layer()
    pre_ev[2].record(main)
    main.wait_stream(side)


pre_ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]


def prereleased_who_waits():
    """Which side is starved when both run ungated: time to the end of the transfer and to the end of the compute."""
    torch.cuda.synchronize()
    pre_ev[0].record(main)
    overlapped_ours_prereleased()
    torch.cuda.synchronize()
    return pre_ev[0].elapsed_time(pre_ev[1]), pre_ev[0].elapsed_time(pre_ev[2])


# reference-style: per layer pointer tables (host-built once here; the reference rebuilds them every call) + K1 launch
ptr_s = [torch.tensor([sb[l].data_ptr() + o * region * nbp + int(b) * region for b in sid.tolist() for o in range(2)], dtype=torch.int64, device="cuda:0") for l in range(nl)]
ptr_d = [torch.tensor([db[l].data_ptr() + o * region * nbp + int(b) * region for b in did.tolist() for o in range(2)], dtype=torch.int64, device="cuda:0") for l in range(nl)]
ref_path = os.path.join(ROOT, "oracle", "_ref", "libkvbm_kernels_ref.so")
R = None
if os.path.exists(ref_path):
    R = C.CDLL(ref_path)
    R.kvbm_kernels_launch_vectorized_copy.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_int, C.c_void_p]
events = [torch.cuda.Event() for _ in range(nl)]


def overlapped_ref_style():
    for l in range(nl):
        compute_layer()
        events[l].record(main)
        side.wait_event(events[l])
        assert R.kvbm_kernels_launch_vectorized_copy(ptr_s[l].data_ptr(), ptr_d[l].data_ptr(), region, 2 * n, sp) == 0
    main.wait_stream(side)


def transfer_only_ref():
    for l in range(nl):
        assert R.kvbm_kernels_launch_vectorized_copy(ptr_s[l].data_ptr(), ptr_d[l].data_ptr(), region, 2 * n, mp) == 0


res = {"standin": a.standin, "gemm_n": a.gemm_n if a.standin == "gemm" else None, "fma_per_16B": a.fma, "standin_blocks": standin_blocks, "ring": [a.warps, a.stages, a.tile], "peer": peer, "layers": nl, "region": region, "blocks": n, "bytes": n * nl * 2 * region, "ctas": a.ctas, "layer_us_target": a.layer_us}
# Round-robin over the modes (one timed pass each per round) so clock / thermal drift hits every mode alike; medians.
modes = {"t_compute_ms": compute_only, "t_compute_plus_signals_ms": compute_and_signal,
         "t_transfer_full_chip_ms": lambda: transfer_only(0), "t_transfer_capped_ms": lambda: transfer_only(a.ctas),
         "t_overlapped_ours_ms": overlapped_ours, "t_overlapped_ours_events_ms": overlapped_ours_events,
         "t_overlapped_ours_prereleased_ms": overlapped_ours_prereleased,
         "t_overlapped_ours_per_layer_ms": overlapped_ours_per_layer}
if R is not None:
    modes["t_transfer_ref_per_layer_ms"] = transfer_only_ref
    modes["t_overlapped_ref_style_ms"] = overlapped_ref_style
samples = {k: [] for k in modes}
for k, fn in modes.items():   # warm every path (and load every kernel) before anything is timed
    fn()
    torch.cuda.synchronize()
for _ in range(a.iters):
    for k, fn in modes.items():
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(main)
        fn()
        e1.record(main)
        torch.cuda.synchronize()
        samples[k].append(e0.elapsed_time(e1))
for k, v in samples.items():
    res[k] = float(np.median(v))
tt, tc = prereleased_who_waits()
res["prereleased_transfer_end_ms"], res["prereleased_compute_end_ms"] = tt, tc
res["slowdown_vs_compute_ours_per_layer"] = res["t_overlapped_ours_per_layer_ms"] / res["t_compute_ms"]
res["slowdown_vs_compute_ours_events"] = res["t_overlapped_ours_events_ms"] / res["t_compute_ms"]
res["hidden_fraction_ours_events"] = (res["t_compute_ms"] + res["t_transfer_capped_ms"] - res["t_overlapped_ours_events_ms"]) / res["t_transfer_capped_ms"]
res["hidden_fraction_ours"] = (res["t_compute_plus_signals_ms"] + res["t_transfer_capped_ms"] - res["t_overlapped_ours_ms"]) / res["t_transfer_capped_ms"]
res["slowdown_vs_compute_ours"] = res["t_overlapped_ours_ms"] / res["t_compute_ms"]
if R is not None:
    res["slowdown_vs_compute_ref_style"] = res["t_overlapped_ref_style_ms"] / res["t_compute_ms"]
torch.cuda.synchronize()
assert done.tolist() == [epoch[0]] * nl, "layer done flags not published"
ok = all(torch.equal(db[l].view(2, nbp, region)[:, did.to(ddev).long()].cpu(), sb[l].view(2, nbp, region)[:, sid.long()].cpu()) for l in (0, nl // 2, nl - 1))
res["bit_exact_probe"] = bool(ok)
print(json.dumps(res, indent=1))
os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
json.dump(res, open(a.out, "w"), indent=1)
