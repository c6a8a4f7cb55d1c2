"""Layer streaming of the layout-transforming hand-offs, timed (kvbm_kernels_paged_permute_gather_streamed,
kvbm_kernels_paged_repage_gather_streamed) against the unstreamed entries.

Shapes (one 4k-token sequence, bf16 unless --cast):
  tp8_tp1   Llama-3-70B KV (80 layers, K/V, 8 heads x 128), page 16: decode rank 0 of TP1 gathers its 8 heads from 8 TP8 ranks;
  tp4_tp2   the same model, decode rank 0 of TP2 gathers 4 heads from 2 TP4 ranks;
  repage    Llama-3-8B KV (32 layers), TP8 page 1 -> TP1 page 16: the re-paging gather of 8 ranks.
Sources are fully contiguous OperationalNHD pools, the destination a fully contiguous UniversalTP pool, random block tables.

gate: every ready flag is set before the launch.  Arms, alternated within each of --iters rounds and timed with CUDA events
      (median): the unstreamed entry, the spinning form at max_ctas 8 / 16 / 32 / the default (half the SMs), and the
      stream-wait form.
tail: a producer stream emulates the prefill: per layer a fixed busy kernel (--layer-us) then the layer's ready flag.  The
      streamed arms are enqueued before the producer; the unstreamed arm waits for the producer's last flag and then launches.
      The spinning form runs at max_ctas 16, 32 and the default.
      Each arm's time is from an event after the last flag to the transfer's end (the exposed tail), median of --iters.
Sample destination blocks of every arm are compared with tests/repage_gather_oracle.py.  One JSON line per arm, with the card's
name and power limit."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
from dynamo_b200 import kernels as K  # noqa: E402
from tests.repage_gather_oracle import repage_gather  # noqa: E402

p = argparse.ArgumentParser()
p.add_argument("--tokens", type=int, default=4096)
p.add_argument("--iters", type=int, default=20)
p.add_argument("--cast", choices=["none", "fp8-to-bf16"], default="none")
p.add_argument("--only", default=None, help="comma-separated shapes: tp8_tp1, tp4_tp2, repage")
p.add_argument("--mode", choices=["gate", "tail", "both"], default="both")
p.add_argument("--layer-us", type=float, default=100.0, help="busy time of one emulated prefill layer (tail mode)")
a = p.parse_args(None if __name__ == "__main__" else [])   # imported: the defaults
CAST = K.CastMode.FP8E4M3_TO_BF16 if a.cast == "fp8-to-bf16" else K.CastMode.NONE
SE, DE = (1, 2) if CAST else (2, 2)
NHD, UTP = int(K.KvBlockLayout.OperationalNHD), int(K.KvBlockLayout.UniversalTP)
torch.cuda.set_device(0)
HD, NO = 128, 2
# name: (layers, source ranks, heads per source rank, source page, destination page)
SHAPES = {"tp8_tp1": (80, 8, 1, 16, 16), "tp4_tp2": (80, 2, 2, 16, 16), "repage": (32, 8, 1, 1, 16)}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    name, _, limit = q.stdout.strip().partition(", ") if q.returncode == 0 else (torch.cuda.get_device_name(0), "", "not read")
    return name, limit


def layer_cycles(us):
    """Clock cycles of a busy kernel that runs `us` microseconds on device 0."""
    props = torch.cuda.get_device_properties(0)
    return int(us * props.clock_rate / 1e3) if hasattr(props, "clock_rate") else int(us * 1980)


def emulate_prefill(prod, flags, nl, epoch, cycles):
    """The prefill on stream `prod`: per layer l a busy kernel of `cycles`, then entry l of every ready-flag array in `flags`."""
    with torch.cuda.stream(prod):
        for l in range(nl):
            torch.cuda._sleep(cycles)
            for f in flags:
                K.check(K.set_flags(f, l, 1, epoch, int(prod.cuda_stream)), "set_flags")


class Pool:
    def __init__(self, nb, nl, page, nh, row, kv):
        self.nb, self.nl, self.kv, self.nh = nb, nl, kv, nh
        self.region = page * nh * row
        self.block = nl * NO * self.region
        self.buf = torch.randint(0, 256, (nb, self.block), dtype=torch.uint8, device="cuda")
        base = self.buf.data_ptr()
        self.layer_base = torch.tensor([base + l * NO * self.region for l in range(nl)], dtype=torch.int64, device="cuda")

    def side(self, ids):
        return K.PermuteSide(K.PagedLayout(self.layer_base.data_ptr(), self.block, self.region, self.region, self.nl, NO, self.nb),
                             ids.data_ptr(), self.kv)


def run_shape(name, nl, ranks, snh, ps, pd):
    T = a.tokens
    ns, nd = -(-T // ps), -(-T // pd)
    srow, drow = HD * SE, HD * DE
    rng = np.random.default_rng(7)
    srcs = [Pool(ns, nl, ps, snh, srow, NHD) for _ in range(ranks)]
    dst = Pool(nd, nl, pd, ranks * snh, drow, UTP)
    init = dst.buf.clone()
    sids = [torch.from_numpy(rng.permutation(ns).astype(np.int32)).cuda() for _ in range(ranks)]
    dids = torch.from_numpy(rng.permutation(nd).astype(np.int32)).cuda()
    windows = [(s, 0, s * snh, snh) for s in range(ranks)]
    ksrcs = [K.PermuteSource(srcs[s].side(sids[s]), snh, 0, s * snh, snh) for s in range(ranks)]
    dside = dst.side(dids)
    ready = torch.zeros((ranks, nl), dtype=torch.int32, device="cuda")
    ws = torch.zeros(K.sync_workspace_words(nl), dtype=torch.int32, device="cuda")
    layer_done = torch.zeros(nl, dtype=torch.int32, device="cuda")
    completion = torch.zeros(1, dtype=torch.int32, device="cuda")
    repage = ps != pd
    stream = torch.cuda.Stream()
    sp = int(stream.cuda_stream)

    def unstreamed(s=sp):
        if repage:
            return K.paged_repage_gather(ksrcs, ps, dside, dst.nh, pd, 0, T, 0, nl, srow, int(CAST), stream=s)
        return K.paged_permute_gather(ksrcs, dside, dst.nh, nd, 0, nl, ps, srow, int(CAST), stream=s)

    def streamed(epoch, mode, ctas, s=sp):
        st = K.PermuteStream()
        for j in range(ranks):
            st.layer_ready_flags[j] = ready[j].data_ptr()
        st.layer_done_flags = layer_done.data_ptr()
        st.epoch = epoch
        st.sync_workspace = ws.data_ptr()
        st.gate_mode = mode
        st.max_ctas = ctas
        st.completion_flag = completion.data_ptr()
        st.completion_value = epoch
        if repage:
            return K.paged_repage_gather_streamed(ksrcs, ps, dside, dst.nh, pd, 0, T, 0, nl, srow, int(CAST), None, st, s)
        return K.paged_permute_gather_streamed(ksrcs, dside, dst.nh, nd, 0, nl, ps, srow, int(CAST), None, st, s)

    # sampled destination blocks against the oracle
    samples = [0, nd // 2, nd - 1]
    src_np = [s.buf.cpu().numpy() for s in srcs]
    sids_np = [x.cpu().numpy() for x in sids]
    init_np = init.cpu().numpy()
    want = {}
    for j in samples:
        tb, te = j * pd, min(T, (j + 1) * pd)
        blocks = [([src_np[s][sids_np[s][b]] for b in range(tb // ps, -(-te // ps))], NHD, snh) for s in range(ranks)]
        d = int(dids[j])
        want[d] = repage_gather(blocks, windows, [init_np[d]], UTP, dst.nh, nl, NO, ps, pd, srow, tb, te, int(CAST))[0]

    def check(arm):
        torch.cuda.synchronize()
        if arm != "unstreamed":
            assert completion.item() & 0xFFFFFFFF == epoch[0], f"{name} {arm}: completion word {completion.item() & 0xFFFFFFFF:#x}, epoch {epoch[0]}"
        got = dst.buf.cpu().numpy()
        for d, w in want.items():
            assert np.array_equal(got[d], w), f"{name} {arm}: destination block {d} differs from the oracle"
        dst.buf.copy_(init)
        torch.cuda.synchronize()

    gpu, limit = card()
    moved = T * nl * NO * dst.nh * drow
    arms = [("unstreamed", None, 0)] + [(f"spin_ctas_{c or 'default'}", K.GATE_SPIN, c) for c in (8, 16, 32, 0)] + \
           [("stream_wait", K.GATE_STREAM_WAIT, 0)]
    epoch = [0]

    def go(arm, s=sp):
        _, mode, ctas = arm
        if mode is None:
            K.check(unstreamed(s), "unstreamed")
        else:
            K.check(streamed(epoch[0], mode, ctas, s), arm[0])

    if a.mode in ("gate", "both"):
        times = {x[0]: [] for x in arms}
        for it in range(a.iters + 2):
            epoch[0] += 1
            ready.fill_(epoch[0])
            torch.cuda.synchronize()
            for arm in arms:
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(stream)
                go(arm)
                e1.record(stream)
                e1.synchronize()
                if it >= 2:
                    times[arm[0]].append(e0.elapsed_time(e1) * 1e3)
                if it == 0:
                    check(arm[0])
        for arm in arms:
            us = statistics.median(times[arm[0]])
            print(json.dumps({"bench": "transform_stream", "mode": "gate", "shape": name, "cast": a.cast, "arm": arm[0], "median_us": round(us, 1),
                              "gb_s": round(moved / us / 1e3, 1), "bytes": moved, "iters": a.iters, "gpu": gpu, "power_limit": limit}), flush=True)

    if a.mode in ("tail", "both"):
        prod = torch.cuda.Stream()
        cycles = layer_cycles(a.layer_us)
        with torch.cuda.stream(prod):   # the producer's kernels load before anything spins
            torch.cuda._sleep(100)
            K.check(K.set_flags(ready[0].data_ptr(), 0, 1, epoch[0], int(prod.cuda_stream)), "set_flags")
        torch.cuda.synchronize()
        tail_arms = [x for x in arms if x[0] in ("unstreamed", "spin_ctas_16", "spin_ctas_32", "spin_ctas_default", "stream_wait")]
        times = {x[0]: [] for x in tail_arms}
        for it in range(a.iters + 2):
            for arm in tail_arms:
                epoch[0] += 1
                torch.cuda.synchronize()
                last = torch.cuda.Event(enable_timing=True)
                end = torch.cuda.Event(enable_timing=True)
                if arm[1] is not None:
                    go(arm)                        # enqueued before the prefill starts
                emulate_prefill(prod, [ready[r].data_ptr() for r in range(ranks)], nl, epoch[0], cycles)
                last.record(prod)
                if arm[1] is None:
                    stream.wait_event(last)
                    go(arm)
                end.record(stream)
                end.synchronize()
                if it >= 2:
                    times[arm[0]].append(last.elapsed_time(end) * 1e3)
                if it == 0:
                    check(arm[0])
        for arm in tail_arms:
            us = statistics.median(times[arm[0]])
            print(json.dumps({"bench": "transform_stream", "mode": "tail", "shape": name, "cast": a.cast, "arm": arm[0],
                              "exposed_tail_us": round(us, 1), "layer_us": a.layer_us, "layers": nl, "iters": a.iters, "gpu": gpu,
                              "power_limit": limit}), flush=True)


if __name__ == "__main__":
    for nm, shape in SHAPES.items():
        if a.only and nm not in a.only.split(","):
            continue
        run_shape(nm, *shape)
        torch.cuda.empty_cache()
