"""Replicate 1 -> N: NVLS multicast (one write per tile, the switch fans it out) vs N unicast bulk stores per tile.

Single process, all visible GPUs; source pool on GPU 0.  Llama-3-8B geometry (32 layers x K/V x 32 KiB regions),
--blocks blocks per transfer.  Timed with CUDA events on the launch stream, medians.  Verifies every receiver pool.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from dynamo_b200 import kernels as K  # noqa: E402
from dynamo_b200.physical import MulticastGroup, TransferManager, multicast_supported  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--blocks", type=int, default=256)
ap.add_argument("--pool", type=int, default=1024)
ap.add_argument("--layers", type=int, default=32)
ap.add_argument("--iters", type=int, default=20)
ap.add_argument("--ctas", type=int, default=0)
ap.add_argument("--modes", default="1,2")
ap.add_argument("--sweep", action="store_true", help="grid over CTAs / warps / stages / tile for the multicast modes (tuning)")
ap.add_argument("--hybrid", action="store_true", help="split the payload: a fraction by multicast, the rest by unicast replicate, concurrently")
ap.add_argument("--out", default="gpurun_out/mc_bench.json")
a = ap.parse_args()

nd = torch.cuda.device_count()
assert nd >= 2 and all(multicast_supported(d) for d in range(nd)), "needs >= 2 GPUs with multicast support"
NL, NO, REGION, NB, n = a.layers, 2, 32768, a.pool, a.blocks
PER_LAYER = NO * NB * REGION
TOTAL = NL * PER_LAYER
torch.cuda.set_device(0)
mgr = TransferManager(device=0)
for d in range(1, nd):
    mgr.enable_peer_access(d)


class _Raw:
    def __init__(self, ptr, nbytes):
        self.__cuda_array_interface__ = {"shape": (nbytes,), "typestr": "|u1", "data": (int(ptr), False), "version": 2}


g = MulticastGroup.create(nd, TOTAL)
for d in range(nd):
    torch.zeros(1, device=f"cuda:{d}")
    g.add_device(d)
pools = []
for d in range(nd):
    with torch.cuda.device(d):
        t = torch.as_tensor(_Raw(g.bind_local(d), TOTAL), device=f"cuda:{d}")
        t.zero_()
        pools.append(t)
for d in range(nd):
    torch.cuda.synchronize(d)
mc = g.map(0)

src = [torch.empty(PER_LAYER, dtype=torch.uint8, device="cuda:0").random_(0, 256) for _ in range(NL)]
sbase = torch.tensor([b.data_ptr() for b in src], dtype=torch.int64, device="cuda:0")
s_desc = K.PagedLayout(sbase.data_ptr(), REGION, REGION * NB, REGION, NL, NO, NB)


def desc_for(base_ptr):
    t = torch.tensor([base_ptr + l * PER_LAYER for l in range(NL)], dtype=torch.int64, device="cuda:0")
    return t, K.PagedLayout(t.data_ptr(), REGION, REGION * NB, REGION, NL, NO, NB)


keep = []
mc_t, mc_desc = desc_for(mc)
uc = []
for d in range(nd):
    t, dsc = desc_for(pools[d].data_ptr())
    keep.append(t)
    uc.append(dsc)
rng = np.random.default_rng(0)
sid = torch.tensor(rng.permutation(NB)[:n], dtype=torch.int32, device="cuda:0")
did = torch.tensor(rng.permutation(NB)[:n], dtype=torch.int32, device="cuda:0")
sp = int(torch.cuda.current_stream().cuda_stream)
payload = n * NL * NO * REGION


def run_mc(mode, ctas=None, warps=0, stages=0, tile=0):
    K.check(K.paged_copy(s_desc, [K.PagedDst(mc_desc, sid.data_ptr(), did.data_ptr(), 0, 0)], n, 0, NL, 0,
                         K.PagedCopyOpts(multicast=mode, max_ctas=a.ctas if ctas is None else ctas, warps_per_cta=warps,
                                         stages=stages, tile_bytes=tile), sp))


def run_unicast(receivers):
    dsts = [K.PagedDst(uc[d], sid.data_ptr(), did.data_ptr(), 0, 0) for d in receivers]
    K.check(K.paged_copy(s_desc, dsts, n, 0, NL, 0, K.PagedCopyOpts(max_ctas=a.ctas), sp))


def t_ms(fn):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(a.iters):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return float(np.median(ts))


def verify(tag, devices=None):
    for d in range(nd):
        torch.cuda.synchronize(d)
    ref = [src[l].view(NO, NB, REGION)[:, sid.long()].cpu() for l in (0, NL - 1)]
    for d in (range(nd) if devices is None else devices):
        for k, l in enumerate((0, NL - 1)):
            got = pools[d][l * PER_LAYER:(l + 1) * PER_LAYER].view(NO, NB, REGION)[:, did.to(pools[d].device).long()].cpu()
            assert torch.equal(got, ref[k]), f"{tag}: pool on cuda:{d} layer {l} differs"
    for p in pools:
        p.zero_()
    for d in range(nd):
        torch.cuda.synchronize(d)


res = {"gpus": nd, "blocks": n, "payload_bytes": payload, "ctas": a.ctas, "group_size": g.size}
for mode, name in ((1, "multicast_st"), (2, "multicast_tma")):
    if str(mode) not in a.modes.split(","):
        continue
    try:
        run_mc(mode)
        verify(name)
        ms = t_ms(lambda: run_mc(mode))
        res[name] = {"ms": ms, "egress_GBps": payload / ms / 1e6, "delivered_GBps": payload * nd / ms / 1e6,
                     "delivered_remote_GBps": payload * (nd - 1) / ms / 1e6}
    except Exception as e:  # noqa: BLE001
        res[name] = {"error": repr(e)}
        print(name, "FAILED", repr(e), flush=True)
        break
    print(name, res[name], flush=True)
if a.sweep:
    res["sweep"] = []
    for mode in (1, 2):
        for ctas in (16, 32, 48, 66, 111, 132):
            for warps, stages, tile in ((4, 6, 16384), (8, 6, 8192), (8, 8, 4096), (4, 12, 8192), (2, 6, 32768), (16, 6, 4096)):
                fn = lambda: run_mc(mode, ctas, warps, stages, tile)  # noqa: E731
                try:
                    ms = t_ms(fn)
                except Exception as e:  # noqa: BLE001
                    print("sweep point failed", mode, ctas, warps, stages, tile, repr(e), flush=True)
                    continue
                row = {"mode": mode, "ctas": ctas, "warps": warps, "stages": stages, "tile": tile, "ms": ms, "egress_GBps": payload / ms / 1e6}
                res["sweep"].append(row)
                print(row, flush=True)
    verify("after sweep")

if a.hybrid:
    # The multicast path tops out at ~403 GB/s of egress whatever the kernel shape (sweep above) while the port carries ~740:
    # send a fraction f of the blocks through the multicast mapping and the rest as unicast replicate, on two streams at once.
    res["hybrid"] = []
    sa, sb = torch.cuda.Stream(device="cuda:0"), torch.cuda.Stream(device="cuda:0")
    recv = list(range(1, nd))[:7]
    for f in (1.0, 0.95, 0.9, 0.85, 0.8, 0.7):
        n_mc = max(1, min(n, int(round(n * f))))
        n_uc = n - n_mc

        def both():
            e0 = torch.cuda.Event(enable_timing=True)
            ea, eb = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(sa)
            sb.wait_event(e0)
            K.check(K.paged_copy(s_desc, [K.PagedDst(mc_desc, sid.data_ptr(), did.data_ptr(), 0, 0)], n_mc, 0, NL, 0,
                                 K.PagedCopyOpts(multicast=1, max_ctas=32), int(sa.cuda_stream)))
            ea.record(sa)
            if n_uc:
                dsts = [K.PagedDst(uc[d], sid[n_mc:].data_ptr(), did[n_mc:].data_ptr(), 0, 0) for d in recv]
                K.check(K.paged_copy(s_desc, dsts, n_uc, 0, NL, 0, K.PagedCopyOpts(max_ctas=64), int(sb.cuda_stream)))
            eb.record(sb)
            torch.cuda.synchronize()
            return max(e0.elapsed_time(ea), e0.elapsed_time(eb))
        for _ in range(3):
            both()
        ms = float(np.median([both() for _ in range(a.iters)]))
        row = {"fraction_multicast": f, "blocks_multicast": n_mc, "blocks_unicast": n_uc, "ms": ms,
               "delivered_remote_GBps": payload * len(recv) / ms / 1e6}
        res["hybrid"].append(row)
        print(row, flush=True)
    verify("after hybrid", devices=recv)
recv = list(range(1, nd))[:7]
run_unicast(recv)
torch.cuda.synchronize()
ms = t_ms(lambda: run_unicast(recv))
res["unicast_replicate"] = {"receivers": len(recv), "ms": ms, "egress_GBps": payload * len(recv) / ms / 1e6,
                            "delivered_remote_GBps": payload * len(recv) / ms / 1e6}
if "ms" in res.get("multicast_st", {}):
    res["speedup_multicast_st_vs_unicast"] = res["unicast_replicate"]["ms"] / res["multicast_st"]["ms"]
print(json.dumps(res, indent=1))
os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
json.dump(res, open(a.out, "w"), indent=1)

# Unbinding a multicast object takes the driver seconds per member; the process is done, so let the driver reclaim it at
# exit instead of paying for the teardown in GPU-box time.
sys.stdout.flush()
os._exit(0)
