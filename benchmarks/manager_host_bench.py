"""Host time per call of the manager's gather entries: how long kvbm_manager_execute_repage_gather and
kvbm_manager_execute_stage_gather hold the calling thread (validation, staging the block tables, the launch), not the transfer.

Llama-3-8B KV geometry (32 layers, K/V, 8 heads x 128, bf16) on fully contiguous device pools, random block tables:
  repage_gather  TP2 -> TP1, 16-token source pages -> 64-token destination pages, tokens 0..1024 (64 source blocks per
                 source, 16 destination blocks)
  stage_gather   PP2 x TP2 -> TP1 (4 windows), 16-token pages, 16 blocks
Each call goes straight to the C entry with arguments built once, timed with a host clock around the call alone; its
notification is waited for outside the timed span, so every call finds a free slot.  Rounds alternate the two entries.
Printed: one JSON line per entry with the median over rounds of each round's median microseconds per call, the rounds'
min-max, and the card's name and power limit read in this run.  Needs a GPU; there is no fallback."""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
from dynamo_b200 import kernels as K  # noqa: E402
from dynamo_b200 import physical as P  # noqa: E402
from dynamo_b200.physical import LayoutConfig, StorageKind, TransferManager  # noqa: E402

p = argparse.ArgumentParser()
p.add_argument("--calls", type=int, default=500, help="timed calls per entry per round")
p.add_argument("--rounds", type=int, default=5)
a = p.parse_args()
if not torch.cuda.is_available():
    sys.exit("manager_host_bench.py needs a GPU")
torch.cuda.set_device(0)
NL, NO, NH, HD = 32, 2, 8, 128
NHD = int(K.KvBlockLayout.OperationalNHD)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    name, _, limit = q.stdout.strip().partition(", ") if q.returncode == 0 else (torch.cuda.get_device_name(0), "", "not read")
    return {"name": name, "power_limit": limit}


mgr = TransferManager(device=0, worker_id=23)
keep = []


def pool(nb, nl, nh, page):
    cfg = LayoutConfig(nb, nl, NO, page, nh * HD, dtype_width_bytes=2, num_heads=nh)
    buf = torch.zeros(cfg.required_bytes(), dtype=torch.uint8, device="cuda")
    keep.append(buf)
    h = mgr.register_fully_contiguous(cfg, buf.data_ptr(), buf.numel(), StorageKind.Device, 0)
    mgr.set_kv_block_layout(h, NHD)
    return h


def ids(n, nb, seed):
    g = torch.Generator().manual_seed(seed)
    x = (C.c_size_t * n)(*torch.randperm(nb, generator=g)[:n].tolist())
    keep.append(x)
    return x


def lists(*arrs):
    x = (C.c_void_p * len(arrs))(*[C.addressof(v) for v in arrs])
    keep.append(x)
    return C.cast(x, C.POINTER(C.POINTER(C.c_size_t)))


opts = P._COptions()
lib = P.lib()
note = C.c_uint64()

# repage_gather: two 4-head sources at 16-token pages into one 8-head destination at 64-token pages
rs = [pool(128, NL, NH // 2, 16) for _ in range(2)]
rd = pool(32, NL, NH, 64)
r_src = lists(ids(64, 128, 1), ids(64, 128, 2))
r_dst = ids(16, 32, 3)
r_win = (P._CHeadWindow * 2)(P._CHeadWindow(0, 0, 0, 4), P._CHeadWindow(1, 0, 4, 4))
r_h = (C.c_uint64 * 2)(*rs)
repage = lambda: lib.kvbm_manager_execute_repage_gather(mgr._h, 2, r_h, r_src, 64, rd, r_dst, 16, 0, 1024, r_win, 2, C.byref(opts),  # noqa: E731
                                                        C.byref(note))

# stage_gather: PP2 x TP2 -> TP1: layers 0..16 from sources 0 and 1, layers 16..32 from sources 2 and 3
ss = [pool(32, NL // 2, NH // 2, 16) for _ in range(4)]
sd = pool(32, NL, NH, 16)
s_src = lists(*[ids(16, 32, 10 + s) for s in range(4)])
s_dst = ids(16, 32, 20)
s_win = (P._CShardWindow * 4)(*[P._CShardWindow(s, 0, 16 * (s // 2), 16, 0, 4 * (s % 2), 4) for s in range(4)])
s_h = (C.c_uint64 * 4)(*ss)
stage = lambda: lib.kvbm_manager_execute_stage_gather(mgr._h, 4, s_h, s_src, sd, s_dst, 16, s_win, 4, None, C.byref(opts),  # noqa: E731
                                                      C.byref(note))


def one_round(call):
    t = []
    for _ in range(a.calls):
        t0 = time.perf_counter_ns()
        rc = call()
        t1 = time.perf_counter_ns()
        if rc != 0:
            sys.exit("call failed: %d %s" % (rc, lib.kvbm_last_error().decode()))
        if lib.kvbm_notification_wait(mgr._h, note.value, 10_000_000) != 0:
            sys.exit("wait failed: " + lib.kvbm_last_error().decode())
        t.append((t1 - t0) / 1e3)
    return statistics.median(t)


def main():
    info = card()
    arms = {"repage_gather": repage, "stage_gather": stage}
    for call in arms.values():       # warm-up: module loads, slots, the first launches
        for _ in range(50):
            call()
            lib.kvbm_notification_wait(mgr._h, note.value, 10_000_000)
    meds = {k: [] for k in arms}
    for _ in range(a.rounds):
        for k, call in arms.items():
            meds[k].append(one_round(call))
    for k, m in meds.items():
        print(json.dumps({"entry": k, "host_us_per_call": round(statistics.median(m), 2), "rounds_min": round(min(m), 2),
                          "rounds_max": round(max(m), 2), "calls_per_round": a.calls, "rounds": a.rounds, "gpu": info["name"],
                          "power_limit": info["power_limit"]}), flush=True)
    torch.cuda.synchronize()
    mgr.close()


if __name__ == "__main__":
    main()
