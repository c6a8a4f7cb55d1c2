"""Writes the SASS of the library's kernels under profiles/ (no GPU needed: cuobjdump reads the sm_90a cubin in the .so).

    python benchmarks/dump_sass.py            -> profiles/sass_<kernel>.txt + profiles/sass_summary.md
The summary counts the mnemonics that show what the kernel is built from: UBLKCP = cp.async.bulk (TMA 1-D bulk),
SYNCS = mbarrier, UTMACMDFLUSH / fences, F2FP = fp8<->bf16 converts, LDG/STG widths for the SIMT kernels."""
import collections
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SO = os.path.join(ROOT, "dynamo_b200", "libkvbm_kernels.so")
# the scaled instantiations (third template argument true) first: the unscaled keys are prefixes of their names
WANT = {"paged_copy_kernelILi1ELb0ELb1": "paged_copy_fp8_to_bf16_scaled", "paged_copy_kernelILi2ELb0ELb1": "paged_copy_bf16_to_fp8_scaled",
        "paged_permute_kernelILi1ELb1ELb1": "paged_permute_fp8_to_bf16_pow2_scaled", "paged_permute_kernelILi1ELb0ELb1": "paged_permute_fp8_to_bf16_mulhi_scaled",
        "paged_permute_kernelILi2ELb1ELb1": "paged_permute_bf16_to_fp8_pow2_scaled", "paged_permute_kernelILi2ELb0ELb1": "paged_permute_bf16_to_fp8_mulhi_scaled",
        "paged_gather_kernelILi1ELb1ELb1": "paged_gather_fp8_to_bf16_pow2_scaled", "paged_gather_kernelILi1ELb0ELb1": "paged_gather_fp8_to_bf16_mulhi_scaled",
        "paged_gather_kernelILi2ELb1ELb1": "paged_gather_bf16_to_fp8_pow2_scaled", "paged_gather_kernelILi2ELb0ELb1": "paged_gather_bf16_to_fp8_mulhi_scaled",
        "paged_copy_kernelILi0": "paged_copy_cast0", "paged_copy_kernelILi1": "paged_copy_fp8_to_bf16", "paged_copy_kernelILi2": "paged_copy_bf16_to_fp8",
        "pair_copy_kernel": "pair_copy_k1", "permute_table_kernelILb1": "permute_table_pow2", "permute_table_kernelILb0": "permute_table_mulhi",
        "paged_permute_kernelILi0ELb1": "paged_permute_pow2", "paged_permute_kernelILi0ELb0": "paged_permute_mulhi",
        "paged_permute_kernelILi1ELb1": "paged_permute_fp8_to_bf16_pow2", "paged_permute_kernelILi1ELb0": "paged_permute_fp8_to_bf16_mulhi",
        "paged_permute_kernelILi2ELb1": "paged_permute_bf16_to_fp8_pow2", "paged_permute_kernelILi2ELb0": "paged_permute_bf16_to_fp8_mulhi",
        "paged_gather_kernelILi0ELb1": "paged_gather_pow2", "paged_gather_kernelILi0ELb0": "paged_gather_mulhi",
        "paged_gather_kernelILi1ELb1": "paged_gather_fp8_to_bf16_pow2", "paged_gather_kernelILi1ELb0": "paged_gather_fp8_to_bf16_mulhi",
        "paged_gather_kernelILi2ELb1": "paged_gather_bf16_to_fp8_pow2", "paged_gather_kernelILi2ELb0": "paged_gather_bf16_to_fp8_mulhi"}
# the re-paging kernel: <cast, row pow2, scaled, small page pow2>, every instantiation named in full (no prefix clashes)
for _c, _cn in ((0, ""), (1, "_fp8_to_bf16"), (2, "_bf16_to_fp8")):
    for _sc in ((0, 1) if _c else (0,)):
        for _r in (1, 0):
            for _p in (1, 0):
                WANT[f"paged_repage_kernelILi{_c}ELb{_r}ELb{_sc}ELb{_p}E"] = (
                    f"paged_repage{_cn}_row_{'pow2' if _r else 'mulhi'}_page_{'pow2' if _p else 'mulhi'}{'_scaled' if _sc else ''}")
                # re-paging with the gather's sources, the same template arguments
                WANT[f"paged_repage_gather_kernelILi{_c}ELb{_r}ELb{_sc}ELb{_p}E"] = (
                    f"paged_repage_gather{_cn}_row_{'pow2' if _r else 'mulhi'}_page_{'pow2' if _p else 'mulhi'}{'_scaled' if _sc else ''}")
                # the layer-streamed (gated, persistent) re-paging gather
                WANT[f"gated_repage_gather_kernelILi{_c}ELb{_r}ELb{_sc}ELb{_p}E"] = (
                    f"gated_repage_gather{_cn}_row_{'pow2' if _r else 'mulhi'}_page_{'pow2' if _p else 'mulhi'}{'_scaled' if _sc else ''}")
                # the same two over a batch of sequences (the unit table)
                WANT[f"paged_batch_repage_gather_kernelILi{_c}ELb{_r}ELb{_sc}ELb{_p}E"] = (
                    f"paged_batch_repage_gather{_cn}_row_{'pow2' if _r else 'mulhi'}_page_{'pow2' if _p else 'mulhi'}{'_scaled' if _sc else ''}")
                WANT[f"gated_batch_repage_gather_kernelILi{_c}ELb{_r}ELb{_sc}ELb{_p}E"] = (
                    f"gated_batch_repage_gather{_cn}_row_{'pow2' if _r else 'mulhi'}_page_{'pow2' if _p else 'mulhi'}{'_scaled' if _sc else ''}")
                # one source into several targets (the gather's mirror image)
                WANT[f"paged_repage_scatter_kernelILi{_c}ELb{_r}ELb{_sc}ELb{_p}E"] = (
                    f"paged_repage_scatter{_cn}_row_{'pow2' if _r else 'mulhi'}_page_{'pow2' if _p else 'mulhi'}{'_scaled' if _sc else ''}")
                # the scatter streamed behind the source's ready flags (gated, persistent)
                WANT[f"gated_repage_push_kernelILi{_c}ELb{_r}ELb{_sc}ELb{_p}E"] = (
                    f"gated_repage_push{_cn}_row_{'pow2' if _r else 'mulhi'}_page_{'pow2' if _p else 'mulhi'}{'_scaled' if _sc else ''}")
                # the routed batch scatter: each sequence to its own targets, one CTA per unit and streamed
                WANT[f"paged_repage_route_kernelILi{_c}ELb{_r}ELb{_sc}ELb{_p}E"] = (
                    f"paged_repage_route{_cn}_row_{'pow2' if _r else 'mulhi'}_page_{'pow2' if _p else 'mulhi'}{'_scaled' if _sc else ''}")
                WANT[f"gated_repage_route_kernelILi{_c}ELb{_r}ELb{_sc}ELb{_p}E"] = (
                    f"gated_repage_route{_cn}_row_{'pow2' if _r else 'mulhi'}_page_{'pow2' if _p else 'mulhi'}{'_scaled' if _sc else ''}")
                # the routed batch gather: each sequence from its own sources, one CTA per unit and streamed
                WANT[f"paged_repage_fanin_kernelILi{_c}ELb{_r}ELb{_sc}ELb{_p}E"] = (
                    f"paged_repage_fanin{_cn}_row_{'pow2' if _r else 'mulhi'}_page_{'pow2' if _p else 'mulhi'}{'_scaled' if _sc else ''}")
                WANT[f"gated_repage_fanin_kernelILi{_c}ELb{_r}ELb{_sc}ELb{_p}E"] = (
                    f"gated_repage_fanin{_cn}_row_{'pow2' if _r else 'mulhi'}_page_{'pow2' if _p else 'mulhi'}{'_scaled' if _sc else ''}")
                # the batch gather between pages that need not divide, one CTA per unit and streamed
                WANT[f"paged_repage_anypage_kernelILi{_c}ELb{_r}ELb{_sc}ELb{_p}E"] = (
                    f"paged_repage_anypage{_cn}_row_{'pow2' if _r else 'mulhi'}_page_{'pow2' if _p else 'mulhi'}{'_scaled' if _sc else ''}")
                WANT[f"gated_repage_anypage_kernelILi{_c}ELb{_r}ELb{_sc}ELb{_p}E"] = (
                    f"gated_repage_anypage{_cn}_row_{'pow2' if _r else 'mulhi'}_page_{'pow2' if _p else 'mulhi'}{'_scaled' if _sc else ''}")
                # the batch scatter between pages that need not divide, one CTA per unit and streamed
                WANT[f"paged_repage_phased_push_kernelILi{_c}ELb{_r}ELb{_sc}ELb{_p}E"] = (
                    f"paged_repage_phased_push{_cn}_row_{'pow2' if _r else 'mulhi'}_page_{'pow2' if _p else 'mulhi'}{'_scaled' if _sc else ''}")
                WANT[f"gated_repage_phased_push_kernelILi{_c}ELb{_r}ELb{_sc}ELb{_p}E"] = (
                    f"gated_repage_phased_push{_cn}_row_{'pow2' if _r else 'mulhi'}_page_{'pow2' if _p else 'mulhi'}{'_scaled' if _sc else ''}")
                # the routed gather and the routed scatter between pages that need not divide, one CTA per unit and streamed
                for _k in ("paged_repage_collect", "gated_repage_collect", "paged_repage_deal", "gated_repage_deal"):
                    WANT[f"{_k}_kernelILi{_c}ELb{_r}ELb{_sc}ELb{_p}E"] = (
                        f"{_k}{_cn}_row_{'pow2' if _r else 'mulhi'}_page_{'pow2' if _p else 'mulhi'}{'_scaled' if _sc else ''}")
            # the layer-streamed (gated, persistent) gather: <cast, row pow2, scaled>
            WANT[f"gated_gather_kernelILi{_c}ELb{_r}ELb{_sc}E"] = f"gated_gather{_cn}_{'pow2' if _r else 'mulhi'}{'_scaled' if _sc else ''}"
WANT["layer_signal_kernel"] = "layer_signal"
WANT["scatter_signal_kernel"] = "scatter_signal"
KEYS = ["UBLKCP.S.G", "UBLKCP.G.S", "SYNCS.ARRIVE.TRANS64", "SYNCS.PHASECHK.TRANS64.TRYWAIT", "SYNCS.ARRIVE", "UTMACMDFLUSH", "FENCE.VIEW.ASYNC",
            "F2FP", "ATOMG", "LDG.E.NA.128", "STG.E.NA.128", "LDS.128", "STS.128", "NANOSLEEP", "SHFL"]


def main():
    txt = subprocess.run(["cuobjdump", "-sass", SO], capture_output=True, text=True, check=True).stdout
    out = os.path.join(ROOT, "profiles")
    os.makedirs(out, exist_ok=True)
    parts = re.split(r"\n\s*Function : ", txt)
    rows = []
    for p in parts[1:]:
        name = p.split("\n", 1)[0].strip()
        tag = next((v for k, v in WANT.items() if k in name), None)
        if not tag:
            continue
        body = p
        ops = collections.Counter(m.group(1) for m in re.finditer(r"^\s*/\*[0-9a-f]+\*/\s+(?:@!?U?P\d\s+)?([A-Z][A-Z0-9_.]+)", body, re.M))
        regs = re.search(r"REG:(\d+)", body)
        with open(os.path.join(out, f"sass_{tag}.txt"), "w") as f:
            f.write("Function : " + p)
        rows.append((tag, name, sum(ops.values()), {k: sum(v for o, v in ops.items() if o.startswith(k)) for k in KEYS}))
    with open(os.path.join(out, "sass_summary.md"), "w") as f:
        f.write("# SASS of the sm_90a kernels in dynamo_b200/libkvbm_kernels.so (`python benchmarks/dump_sass.py`)\n\n")
        f.write("| kernel | instructions | " + " | ".join(KEYS) + " |\n|---|---:|" + "---:|" * len(KEYS) + "\n")
        for tag, name, total, c in rows:
            f.write(f"| `{tag}` | {total} | " + " | ".join(str(c[k]) for k in KEYS) + " |\n")
        f.write("\nUBLKCP.S.G / UBLKCP.G.S = cp.async.bulk global->shared / shared->global (TMA 1-D bulk copies); SYNCS.* = mbarrier "
                "arrive / expect_tx / try_wait; F2FP = e4m3<->f16/f32 converts of the fused cast; the K1 and permute kernels are SIMT "
                "(128-bit LDG/STG with L1 no-allocate).\n")
    for r in rows:
        print(r[0], r[2], {k: v for k, v in r[3].items() if v})


if __name__ == "__main__":
    main()
