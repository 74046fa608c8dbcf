#!/usr/bin/env python
"""Sweep of the tiled passes of K1p (spmm_panel.cu) against the one-pass kernel; prints one JSON line.

At C2 (CSR 1e6 x 1e6, nnz 1e8, B 1e6 x 128 fp32): panel budgets x tile widths, the all-hit ceiling (same shape and nnz,
every column inside one 16 MB panel, so every gather after the first touch of a line is an L2 hit), evict_last
against no L2 hint on the B loads, and shapes on both sides of the automatic choice (one-pass, automatic, and the
passes forced at the default panel budget).  Every timed result is compared
bit for bit with the one-pass kernel.  Next to each time: the DRAM-byte model of the path (computed from shapes, not
measured).  Run from the repository root: python tools/tune_panels.py
"""
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from sparse_b200 import _kernels as Kn  # noqa: E402
from sparse_b200 import _lib  # noqa: E402
from tools.tune_k1 import timeit  # noqa: E402

MB = 1 << 20
L2_DEFAULT = 50 * MB


def dram_model(M, K, N, nnz, es, ib, tile_bytes, P):
    """Bytes the tiled path moves through HBM if every gather after the first touch hits L2: C (2P-1) x per tile,
    A once per tile, B once, the offsets pre-pass (indices read, (P+1) x M offsets written) and the offsets reads."""
    row = N * es
    tiles = -(-row // tile_bytes)
    c = M * row * (2 * P - 1)
    a = tiles * nnz * (es + ib)
    b = K * row
    pre = nnz * ib + (P + 1) * M * ib
    offs = tiles * P * 2 * M * ib
    return {"C": c, "A": a, "B": b, "prepass": pre, "offsets": offs, "total_GB": round((c + a + b + pre + offs) / 1e9, 2)}


def panels_of(K, N, es, panel_bytes, tile_bytes):
    tb = min(tile_bytes, max(64, 1 << (N * es - 1).bit_length()))
    return max(1, -(-K * tb // panel_bytes)), tb


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30)
        return r.stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"unavailable ({e})"


def csr(M, K, nnz, seed, dev, col_hi=None):
    vals, cols, indptr, _ = bench.gen_A(torch, M, col_hi or K, nnz, seed, dev)
    return vals, cols, indptr


def run(vals, cols, indptr, B, M, K, N, C, n_panels):
    return lambda: Kn.spmm_csr_dense(vals, cols, indptr, B, M, K, N, out=C, n_panels=n_panels)


def launches(fn):
    n0 = _lib.launch_count()
    fn()
    torch.cuda.synchronize()
    return _lib.launch_count() - n0


def main():
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    out = {"card": card()}
    M = K = 1_000_000
    nnz = 100_000_000
    vals, cols, indptr = csr(M, K, nnz, 1234, dev)
    B = bench.gen_B(torch, K, 128, 99, dev)
    C = torch.empty((M, 128), dtype=torch.float32, device=dev)
    alg = bench.algorithmic_bytes(nnz, M, 128)

    Kn.spmm_set_tiling(0, 0)
    one = run(vals, cols, indptr, B, M, K, 128, C, 1)
    ms1 = timeit(one)
    ref = C.clone()
    out["c2_one_pass"] = {"ms": round(ms1, 3), "gather_model_GB": round(alg / 1e9, 2)}

    sweep = []
    for tb in (64, 128, 256):
        for pmb in (8, 12, 16, 24, 32, 48):
            Kn.spmm_set_tiling(pmb * MB, tb)
            P, tbe = panels_of(K, 128, 4, pmb * MB, tb)
            ms = timeit(run(vals, cols, indptr, B, M, K, 128, C, 0))
            sweep.append({"panel_MB": pmb, "tile_B": tb, "P": P, "ms": round(ms, 3), "vs_one_pass": round(ms / ms1, 3),
                          "bit_equal": bool(torch.equal(C, ref)),
                          "dram_model_GB": dram_model(M, K, 128, nnz, 4, 4, tbe, P)["total_GB"]})
            print(sweep[-1], file=sys.stderr, flush=True)
    out["c2_sweep"] = sweep
    Kn.spmm_set_tiling(0, 0)

    # evict_last vs no hint on the B loads (default tiling)
    auto = run(vals, cols, indptr, B, M, K, 128, C, 0)
    ms_hint = timeit(auto)
    Kn.spmm_set_variant(4, 8)
    ms_nohint = timeit(auto)
    eq = bool(torch.equal(C, ref))
    Kn.spmm_set_variant(1, 8)
    out["c2_b_hint"] = {"evict_last_ms": round(ms_hint, 3), "no_hint_ms": round(ms_nohint, 3), "bit_equal": eq}
    print(out["c2_b_hint"], file=sys.stderr, flush=True)
    del vals, cols, indptr

    # all-hit ceiling: same shape and nnz, columns only in the first 16 MB panel of a 128-byte tile
    hi = 16 * MB // 128
    v2, c2, p2 = csr(M, K, nnz, 4321, dev, col_hi=hi)
    Kn.spmm_set_tiling(16 * MB, 128)
    ms_ceil = timeit(run(v2, c2, p2, B, M, K, 128, C, 0))
    r2 = C.clone()
    ms_ceil1 = timeit(run(v2, c2, p2, B, M, K, 128, C, 1))
    out["all_hit_ceiling"] = {"col_range": hi, "P": 8, "tiled_ms": round(ms_ceil, 3), "one_pass_ms": round(ms_ceil1, 3),
                              "bit_equal": bool(torch.equal(C, r2)), "gathers_per_s_G": round(nnz * 4 / ms_ceil / 1e6, 2),
                              "dram_model_GB": dram_model(M, K, 128, nnz, 4, 4, 128, 8)["total_GB"]}
    print(out["all_hit_ceiling"], file=sys.stderr, flush=True)
    Kn.spmm_set_tiling(0, 0)
    del v2, c2, p2

    # shapes around the thresholds: automatic choice vs the one-pass kernel
    shapes = []
    cases = [(1_000_000, 1_000_000, 10_000_000, 128, torch.float32), (1_000_000, 1_000_000, 30_000_000, 128, torch.float32),
             (1_000_000, 1_000_000, 50_000_000, 128, torch.float32), (1_000_000, 1_000_000, 70_000_000, 128, torch.float32),
             (1_000_000, 100_000, 10_000_000, 128, torch.float32), (1_000_000, 100_000, 30_000_000, 128, torch.float32),
             (1_000_000, 1_000_000, 100_000_000, 64, torch.float32),
             (1_000_000, 1_000_000, 100_000_000, 256, torch.float32),
             (1_000_000, 1_000_000, 100_000_000, 64, torch.float64)]
    for (m, k, z, n, dt) in cases:
        v, c, p = csr(m, k, z, 777, dev)
        v = v.to(dt)
        Bn = bench.gen_B(torch, k, n, 5, dev).to(dt)
        Cn = torch.empty((m, n), dtype=dt, device=dev)
        t1 = timeit(run(v, c, p, Bn, m, k, n, Cn, 1))
        rr = Cn.clone()
        fa = run(v, c, p, Bn, m, k, n, Cn, 0)
        ta = timeit(fa)
        es = torch.finfo(dt).bits // 8
        n_l = launches(fa)
        eq = bool(torch.equal(Cn, rr))
        P, tbe = panels_of(k, n, es, 24 * MB, 128)
        # the passes forced at the default panel budget (at least 2 panels), whichever side of the thresholds
        tt = timeit(run(v, c, p, Bn, m, k, n, Cn, max(2, P)))
        shapes.append({"M": m, "K": k, "nnz": int(v.numel()), "N": n, "dtype": str(dt).replace("torch.", ""),
                       "one_pass_ms": round(t1, 3), "auto_ms": round(ta, 3), "auto_launches": n_l,
                       "auto_is_tiled": n_l > 3, "tiled_ms": round(tt, 3), "tiled_P": max(2, P),
                       "bit_equal": eq and bool(torch.equal(Cn, rr)),
                       "gather_model_GB": round(bench.algorithmic_bytes(int(v.numel()), m, n) * es / 4 / 1e9, 2),
                       "tiled_dram_model_GB": dram_model(m, k, n, int(v.numel()), es, 4, tbe, P)["total_GB"]})
        print(shapes[-1], file=sys.stderr, flush=True)
        del v, c, p, Bn, Cn, rr
        torch.cuda.empty_cache()
    out["shapes"] = shapes
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
