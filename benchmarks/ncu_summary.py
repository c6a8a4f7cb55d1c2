"""Summarises .ncu-rep captures (read here, no GPU needed) into a small JSON + markdown table for profiles/.

    python benchmarks/ncu_summary.py prof_ours.ncu-rep [more.ncu-rep ...] --out profiles/ncu_summary
"""
import argparse
import csv
import io
import json
import subprocess

KEYS = {
    "gpu__time_duration.sum": "duration_ns",
    "dram__bytes_read.sum": "dram_read_bytes",
    "dram__bytes_write.sum": "dram_write_bytes",
    "dram__throughput.avg.pct_of_peak_sustained_elapsed": "dram_pct_peak",
    "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed": "gpu_dram_pct_peak",
    "lts__t_sector_hit_rate.pct": "l2_hit_rate_pct",
    "lts__t_bytes.sum": "l2_bytes",
    "sm__throughput.avg.pct_of_peak_sustained_elapsed": "sm_pct_peak",
    "sm__warps_active.avg.pct_of_peak_sustained_active": "achieved_occupancy_pct",
    "launch__registers_per_thread": "registers_per_thread",
    "launch__grid_size": "grid",
    "launch__block_size": "block",
    "launch__shared_mem_per_block_dynamic": "dyn_smem_bytes",
    "smsp__cycles_active.avg": "smsp_cycles_active",
    "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active": "tensor_pipe_pct",
    "l1tex__m_xbar2l1tex_read_bytes.sum": "l1_fill_bytes",
    "nvltx__bytes.sum": "nvlink_tx_bytes",
    "nvlrx__bytes.sum": "nvlink_rx_bytes",
    "smsp__average_warp_latency_issue_stalled_long_scoreboard.ratio": "stall_long_scoreboard",
    "smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio": "stall_long_scoreboard_per_issue",
}


def rows(path):
    out = subprocess.run(["ncu", "-i", path, "--page", "raw", "--csv"], capture_output=True, text=True, check=True).stdout
    rd = list(csv.reader(io.StringIO(out)))
    hdr, units, data = rd[0], rd[1], rd[2:]
    res = []
    for r in data:
        d = dict(zip(hdr, r))
        item = {"kernel": d.get("Kernel Name", "?")[:90], "id": d.get("ID")}
        for k, name in KEYS.items():
            if k in d and d[k] != "":
                try:
                    v = float(d[k].replace(",", ""))
                except ValueError:
                    continue
                u = units[hdr.index(k)]
                if name.endswith("_bytes") or name == "l2_bytes":
                    mult = {"byte": 1, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9, "Tbyte": 1e12}.get(u, 1)
                    v *= mult
                if name == "duration_ns":
                    v *= {"ns": 1, "us": 1e3, "usecond": 1e3, "ms": 1e6, "msecond": 1e6, "nsecond": 1, "s": 1e9, "second": 1e9}.get(u, 1)
                item[name] = v
        if "dram_read_bytes" in item and "dram_write_bytes" in item and "duration_ns" in item:
            item["dram_total_bytes"] = item["dram_read_bytes"] + item["dram_write_bytes"]
            item["dram_gbs"] = item["dram_total_bytes"] / item["duration_ns"]
        res.append(item)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("reps", nargs="+")
    ap.add_argument("--out", default="profiles/ncu_summary")
    a = ap.parse_args()
    allr = {}
    md = ["| capture | kernel | dur (us) | DRAM rd (MB) | DRAM wr (MB) | DRAM GB/s | DRAM % peak | L2 hit % | regs | grid x block | smem |",
          "|---|---|---:|---:|---:|---:|---:|---:|---:|---|---:|"]
    for p in a.reps:
        try:
            r = rows(p)
        except Exception as e:  # noqa
            print("failed", p, e)
            continue
        allr[p] = r
        for it in r:
            md.append("| %s | %s | %.1f | %.1f | %.1f | %.0f | %.1f | %.1f | %d | %dx%d | %d |" % (
                p.split("/")[-1], it["kernel"][:48], it.get("duration_ns", 0) / 1e3, it.get("dram_read_bytes", 0) / 1e6,
                it.get("dram_write_bytes", 0) / 1e6, it.get("dram_gbs", 0), it.get("dram_pct_peak", it.get("gpu_dram_pct_peak", 0)),
                it.get("l2_hit_rate_pct", 0), it.get("registers_per_thread", 0), it.get("grid", 0), it.get("block", 0),
                it.get("dyn_smem_bytes", 0)))
    json.dump(allr, open(a.out + ".json", "w"), indent=1)
    open(a.out + ".md", "w").write("\n".join(md) + "\n")
    print("\n".join(md))


if __name__ == "__main__":
    main()
