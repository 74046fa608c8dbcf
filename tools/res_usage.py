#!/usr/bin/env python
"""Static resource usage of the hot-path kernels (registers, stack = spills, static shared memory) from
`cuobjdump -res-usage` of the in-tree library -- no GPU needed.  Writes a markdown table (stdout).

    python tools/res_usage.py > res_usage.md
"""
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "sparse_b200", "libsparse_b200.so")
# the instantiations the benchmark configurations launch (fp32 / fp64 values, int32 / int64 indices)
HOT = [r"spmm_csr_dense_dyn_kernel<float, int, 4, 32, 8, 4>", r"spmm_csr_dense_dyn_kernel<float, int, 4, 32, 8, 5>",
       r"spmm_csr_dense_kernel<float, int, 4, 32, 8", r"spmm_tile_pass_kernel<float, int, 8>",
       r"spmm_long_rows_ring_kernel<float", r"spgemm_products_kernel", r"spgemm_rows_kernel<float",
       r"spgemm_rows_kernel<double", r"spgemm_block_kernel<float", r"spgemm_finish_kernel<float",
       r"ew_merge_kernel<double", r"ew_merge_kernel<float", r"rd_count_kernel", r"rd_emit_kernel<double",
       r"rd_emit_kernel<float", r"reduce_tile_kernel<double", r"sddmm_kernel<float", r"mttkrp_kernel<float", r"mttkrp_mode_kernel<float", r"mttkrp_combine_kernel<float",
       r"ttmc_mode_kernel<float, int, 4, 16, 8>", r"ttmc_mode_kernel<float, int, 1, 16, 8>",
       r"ttmc_mode_kernel<double, int, 2, 16, 8>", r"tttp_kernel<float, int, 4>", r"tttp_kernel<float, int, 1>",
       r"tttp_kernel<double, int, 2>", r"ttm_mode_kernel<float, int, 4>", r"ttm_mode_kernel<float, int, 1>",
       r"ttm_mode_kernel<double, int, 2>", r"cp_completion_kernel<float, int, 4, 4>",
       r"cp_completion_kernel<float, int, 4, 9>", r"cp_completion_kernel<double, int, 2, 9>",
       r"cp_completion_combine_kernel<float, int>", r"cp_apr_phi_kernel<float, int, 4, 4, 4, 4>",
       r"cp_apr_phi_kernel<float, int, 4, 8, 4, 4>", r"cp_apr_phi_kernel<double, int, 2, 32, 2, 8>",
       r"masked_spgemm_kernel<float, float, int, 32>", r"masked_spgemm_kernel<double, double, int, 8>",
       r"spmm_bulk_kernel<float"]


def main():
    out = subprocess.run(["cuobjdump", "-res-usage", LIB], capture_output=True, text=True, check=True).stdout
    rows, name = [], None
    for line in out.splitlines():
        m = re.match(r"\s*Function (\S+):", line)
        if m:
            name = m.group(1)
            continue
        m = re.search(r"REG:(\d+) STACK:(\d+) SHARED:(\d+) LOCAL:(\d+)", line)
        if m and name:
            rows.append((name,) + tuple(int(v) for v in m.groups()))
            name = None
    dem = subprocess.run(["c++filt"], input="\n".join(r[0] for r in rows), capture_output=True, text=True).stdout.splitlines()
    rows = [(d,) + r[1:] for d, r in zip(dem, rows)]
    print("# Static resource usage of the hot-path kernels (`cuobjdump -res-usage sparse_b200/libsparse_b200.so`, sm_90a)\n")
    print(f"{len(rows)} kernels in the library; kernels with a non-zero stack (spill) frame: "
          f"{sum(1 for r in rows if r[2] > 0)}; maximum registers per thread: {max(r[1] for r in rows)}.\n")
    print("Dynamic shared memory (the ring buffers of the long-row SpMM kernel, the per-warp hash tables of SpGEMM, the "
          "merge tiles of the element-wise kernel) is requested at launch and is not part of `SHARED` below.\n")
    print("| kernel (the instantiation the C2 / C5 / C3 / C4 configurations launch; the 5-CTA K1 form is a tuning variant) | registers | stack bytes | static shared bytes | local bytes |")
    print("|---|---|---|---|---|")
    for pat in HOT:
        hit = [r for r in rows if pat in r[0].replace("b2s::", "")]
        if not hit:
            continue
        r = hit[0]
        short = re.sub(r"\(.*", "", r[0].replace("void b2s::", "").replace("b2s::", ""))
        print(f"| `{short}` | {r[1]} | {r[2]} | {r[3]} | {r[4]} |")
    spills = sorted((r for r in rows if r[2] > 0), key=lambda r: -r[2])[:12]
    if spills:
        print("\nKernels with a stack frame (largest first):\n")
        for r in spills:
            print(f"* `{re.sub(r'\(.*', '', r[0].replace('void b2s::', ''))[:140]}`: {r[2]} B stack, {r[1]} registers")
    return 0


if __name__ == "__main__":
    sys.exit(main())
