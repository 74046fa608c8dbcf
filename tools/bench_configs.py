#!/usr/bin/env python
"""Time (and parity-check against the oracle / the reference's digests) the non-headline BASELINE.json configs (C1, C3, C4, C5, reductions, MTTKRP) through the public API.

Device-resident inputs (generated with seeded torch generators on the GPU), wall-clock around
torch.cuda.synchronize() because the public calls contain their own size-returning syncs.
Prints one line per config as it runs and the whole result as one JSON line at the end.

    python tools/bench_configs.py [c1 c3 c3big red c4 c5 mttkrp mttkrp_mode masked ttmc tttp ttm completion cp_apr sptc]

`masked` (the masked SpGEMM, examples/triangles_example.py), `ttmc` (the Tucker / HOOI step), `tttp` (a CP model at
a sparse tensor's entries), `ttm` (mode-n tensor times matrix with a sparse result), `completion` (the ALS update
of CP tensor completion), `cp_apr` (the ratio MTTKRP of Poisson CP) and `sptc` (sparse x sparse tensor contraction on
compressed rows) run only when named.
"""
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
import sparse_b200 as sp  # noqa: E402
from sparse_b200 import _lib  # noqa: E402

DEV = torch.device("cuda", torch.cuda.current_device() if torch.cuda.is_available() else 0)
PEAK, _ = bench.peaks()


def timeit(fn, reps=5, warm=2):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append((time.perf_counter() - t0) * 1e3)
    return min(ts), float(np.median(ts))


def rand_coo(shape, nnz, seed, dtype=torch.float64):
    g = torch.Generator(device=DEV).manual_seed(seed)
    size = int(np.prod(shape))
    lin = torch.unique(torch.randint(0, size, (int(nnz * 1.02) + 64,), generator=g, device=DEV, dtype=torch.int64))
    if lin.numel() > nnz:
        lin = lin[torch.randperm(lin.numel(), generator=g, device=DEV)[:nnz]].sort().values
    coords = torch.stack(torch.unravel_index(lin, shape))
    data = torch.rand(lin.numel(), generator=g, device=DEV, dtype=dtype)
    return sp.COO(coords, data, shape=shape, has_duplicates=False, sorted=True)


def rand_csr(M, K, nnz, seed, dtype=torch.float32):
    vals, cols, indptr, _ = bench.make_workload(torch, M, K, nnz, 1, seed, DEV)
    return sp.GCXS((vals.to(dtype), cols, indptr), shape=(M, K), compressed_axes=(0,))


def run(which=None, compact=False, parity=True):
    """Time the configs; returns {name: {ms_best, ..., frac_of_hbm_peak, parity}}.  `compact` = the subset bench.py
    embeds in its JSON line (one entry per BASELINE.json config + reductions + MTTKRP)."""
    import oracle  # the checker (tests / bench only)

    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    import fullsize_inputs as FI

    which = which or ["c1", "c3", "red", "c5", "c4", "mttkrp", "mttkrp_mode", "c3big"]
    res = {}
    _lib.load()

    def rec(name, fn, units, unit_name, alg_bytes=None, reps=5):
        n0 = _lib.launch_count()
        fn()
        launches = _lib.launch_count() - n0
        best, med = timeit(fn, reps=reps)
        r = {"ms_best": round(best, 4), "ms_median": round(med, 4), unit_name: round(units / best / 1e6, 4),
             "launches_per_call": int(launches)}
        if alg_bytes:
            r["alg_GBs"] = round(alg_bytes / best / 1e6, 1)
            r["frac_of_hbm_peak"] = round(alg_bytes / best / 1e6 / PEAK, 4)
        res[name] = r
        if not compact:
            print(name, r, flush=True)
        return r

    if "c1" in which:
        rng = np.random.default_rng(42)
        a = sp.random((1000, 1000), density=0.01, random_state=rng)
        b = sp.random((1000, 1000), density=0.01, random_state=rng)
        a._dev(); b._dev()
        bd = b.todense()
        out = sp.tensordot(a, b, axes=1)
        r = rec("C1 COO(1000^2@.01) . COO -> COO (f64)", lambda: sp.tensordot(a, b, axes=1), 1e5,
                "Mproducts_per_ms_x1e-3")
        r["out_nnz"] = out.nnz
        if parity:
            ip_a = np.searchsorted(a.coords[0], np.arange(1001))
            ip_b = np.searchsorted(b.coords[0], np.arange(1001))
            co, d = oracle.dot_coo_coo((1000, 1000), a.coords, b.coords, a.data, b.data, ip_a, ip_b)
            order = np.lexsort((co[1], co[0]))
            r["parity"] = {"vs": "oracle _dot_coo_coo + canonical sort", "coords_exact": bool(
                np.array_equal(out.coords, co[:, order])), "data_bit_exact": bool(
                np.array_equal(out.data.view(np.uint64), d[order].view(np.uint64)))}
        if not compact:
            bdev = torch.from_numpy(bd).to(DEV)
            rec("C1 COO . dense -> dense (device operand)", lambda: sp.tensordot(a, bdev, axes=1), a.nnz * 1000,
                "Gmadd_s")

    if "c3" in which or "red" in which:
        (ca, da), (cb, db) = FI.c3_inputs(np.float64)
        a = sp.COO(ca, da, shape=FI.C3_SHAPE_A, has_duplicates=False, sorted=True)
        b = sp.COO(cb, db, shape=FI.C3_SHAPE_B, has_duplicates=False, sorted=True)
        a._dev(); b._dev()
        want = {}
        try:
            with open(os.path.join(ROOT, "tests", "golden", "fullsize_digests.json")) as f:
                want = json.load(f)["cases"]
        except OSError:
            pass
        if "c3" in which:
            out = a + b
            alg = (a.nnz + b.nnz) * 16 + out.nnz * (32 + 8)
            r = rec("C3 COO add (512,512,512,64)+(512,512,512,1) f64", lambda: a + b, a.nnz + b.nnz, "Gnnz_in_s", alg)
            r["out_nnz"] = out.nnz
            if parity and want:
                w = want["c3_add_float64"]
                r["parity"] = {"vs": "the reference's own result (SHA-256 of coords + value bits, "
                                     "tests/golden/fullsize_digests.json)",
                               "nnz_equal": bool(out.nnz == w["nnz"]),
                               "digest_equal": bool(FI.coo_digest(out.coords, out.data) == w["sha256"])}
            if not compact:
                rec("C3 multiply (same operands)", lambda: a * b, a.nnz + b.nnz, "Gnnz_in_s")
        if "red" in which:
            for name, axis in (("reduce sum axis=3", (3,)), ("reduce sum axis=(0,1)", (0, 1)),
                               ("reduce max axis=0", (0,))):
                red = "max" if "max" in name else "sum"
                r = rec(name + " (C3 tensor)", lambda: getattr(a, red)(axis=axis), a.nnz, "Gnnz_s", a.nnz * 16)
                key = f"c3_{red}_axis{''.join(map(str, axis))}_float64"
                if parity and key in want:
                    got = getattr(a, red)(axis=axis)
                    w = want[key]
                    r["parity"] = {"vs": "the reference's own result (coords digest + sampled values, rtol 1e-12)",
                                   "coords_equal": bool(got.nnz == w["nnz"] and FI.digest(
                                       np.asarray(got.coords, dtype=np.int64)) == w["coords_sha256"]),
                                   "values_close": bool(np.allclose(got.data[:: w["sample_step"]], w["values_sample"],
                                                                    rtol=1e-12, atol=0))}
        del a, b

    if "c3big" in which:
        a = rand_coo((512, 512, 512, 64), 85_899_345, 10)
        b = rand_coo((512, 512, 512, 1), 1_342_177, 11)
        out = a + b
        alg = (a.nnz + b.nnz) * 16 + out.nnz * (32 + 8)
        r = rec("C3-large add density 1e-2 (8.6e7 nnz) f64", lambda: a + b, a.nnz + b.nnz, "Gnnz_in_s", alg, reps=3)
        r["out_nnz"] = out.nnz
        if parity:
            # size-independent properties: |union| = |a| + 64|b| - |matches|, every matched position holds a + b,
            # and the value total is the sum of the operands' totals (fp64, tolerance)
            ka, kb = a.sorted_keys(), b.sorted_keys()
            hit = torch.isin(torch.div(ka, 64, rounding_mode="floor"), kb)
            n_match = int(hit.sum().item())
            tot = float(out._data_dev().sum().item())
            exp = float(a._data_dev().sum().item()) + 64.0 * float(b._data_dev().sum().item())
            ko = out.sorted_keys()
            r["parity"] = {"vs": "properties (union size, strictly increasing keys, total)",
                           "union_size": bool(out.nnz == a.nnz + 64 * b.nnz - n_match),
                           "keys_strictly_increasing": bool((ko[1:] > ko[:-1]).all().item()),
                           "total_close": bool(abs(tot - exp) <= 1e-9 * abs(exp))}
            del ka, kb, hit, ko
        del out
        r = rec("reduce-large sum axis=3 (8.6e7 nnz)", lambda: a.sum(axis=3), a.nnz, "Gnnz_s", a.nnz * 16, reps=3)
        if parity:
            got = a.sum(axis=3)
            gk = torch.unique_consecutive(torch.div(a.sorted_keys(), 64, rounding_mode="floor"))
            tot, exp = float(got._data_dev().sum().item()), float(a._data_dev().sum().item())
            r["parity"] = {"vs": "properties (group ids = distinct key // 64, total)",
                           "groups_equal": bool(got.nnz == gk.numel() and torch.equal(got.sorted_keys(), gk)),
                           "total_close": bool(abs(tot - exp) <= 1e-9 * abs(exp))}
            del got, gk
        del a, b

    if "c5" in which:
        for dt, name in ((torch.float32, "f32"), (torch.float64, "f64")):
            if compact and name == "f64":
                continue
            A = rand_csr(1_000_000, 1_000_000, 10_000_000, 3, dt)
            out = sp.tensordot(A, A, axes=1)
            vb = 4 if dt == torch.float32 else 8
            alg = A.nnz * (vb + 4) + 4e6 + 1e8 * (vb + 4) + out.nnz * (vb + 8) + 8e6
            r = rec(f"C5 CSR(1e6^2@1e-5)^2 {name}", lambda: sp.tensordot(A, A, axes=1), out.nnz, "Gnnz_out_s", alg,
                    reps=3)
            r["out_nnz"] = out.nnz
            if parity:
                # rows are independent: the first 20000 rows of the product against the oracle's _dot_csr_csr
                # (reverse-first-touch column order, then prune) on the same arrays
                rows = 20_000
                ad, ai, ap = A.data, A.indices.astype(np.int64), A.indptr.astype(np.int64)
                n = int(ap[rows])
                d, i, p = oracle.dot_csr_csr((rows, 1_000_000), ad[:n], ad, ai[:n], ai, ap[: rows + 1], ap)
                keep = d.view(np.uint32 if vb == 4 else np.uint64) != 0
                m = int(out.indptr[rows])
                r["parity"] = {"vs": f"oracle _dot_csr_csr on the first {rows} rows (all of B)",
                               "indices_exact": bool(m == int(keep.sum()) and np.array_equal(out.indices[:m], i[keep])),
                               "data_bit_exact": bool(m == int(keep.sum()) and np.array_equal(
                                   out.data[:m].view(np.uint8), d[keep].view(np.uint8)))}
            del A, out

    if "c4" in which:
        M = N = 1_000_000
        K = 256
        nnz = 100_000_000
        vals, cols, indptr, _ = bench.make_workload(torch, M, N, nnz, 1, 21, DEV)
        S = sp.GCXS((vals, cols, indptr), shape=(M, N), compressed_axes=(0,)).tocoo()
        g = torch.Generator(device=DEV).manual_seed(22)
        A = torch.rand((M, K), generator=g, device=DEV, dtype=torch.float32)
        B = torch.rand((K, N), generator=g, device=DEV, dtype=torch.float32)
        from sparse_b200 import _kernels as Kn
        from sparse_b200._dot import _coo_as_csr
        sv, sc, sip = _coo_as_csr(S, np.float32)
        Bt = Kn.transpose_dense(B)
        alg = nnz * 12 + M * K * 4 + nnz * K * 4 + nnz * 4
        r = rec("C4 SDDMM kernel only (1e6^2 mask nnz=1e8, K=256 f32)", lambda: Kn.sddmm(sip, sc, sv, A, Bt, M, N, K),
                nnz, "Gnnz_s", alg, reps=5)
        if parity:
            ov = Kn.sddmm(sip, sc, sv, A, Bt, M, N, K)
            gsel = torch.Generator(device=DEV).manual_seed(23)
            sel = torch.randint(0, nnz, (4096,), generator=gsel, device=DEV)
            rows_of = torch.searchsorted(sip.to(torch.int64), sel, right=True) - 1
            dots = (A[rows_of].double() * Bt[sc[sel].to(torch.int64)].double()).sum(dim=1)  # fp64 restatement
            wantv = sv[sel].double() * dots
            r["parity"] = {"vs": "fp64 restatement of s * dot(A[i,:], B[:,j]) on 4096 sampled entries, rtol 2e-5",
                           "values_close": bool(torch.allclose(ov[sel].double(), wantv, rtol=2e-5, atol=0))}
            del ov
        if not compact:
            rec("C4 SDDMM public sddmm(s,a,b) incl. B transpose + prune", lambda: sp.sddmm(S, A, B), nnz, "Gnnz_s",
                alg, reps=3)
        del S, A, B, Bt, sv, sc, sip, vals, cols, indptr

    if "mttkrp" in which:
        I_, K_, L_, J = 10_000, 10_000, 1_000, 32
        Bt = rand_coo((I_, K_, L_), 10_000_000, 31, torch.float32)
        g = torch.Generator(device=DEV).manual_seed(32)
        Dm = torch.rand((L_, J), generator=g, device=DEV, dtype=torch.float32)
        Cm = torch.rand((K_, J), generator=g, device=DEV, dtype=torch.float32)
        alg = Bt.nnz * 16 + 2 * Bt.nnz * J * 4 + I_ * J * 4
        r = rec("MTTKRP fused (1e4 x 1e4 x 1e3, nnz 1e7, J=32 f32)", lambda: sp.mttkrp(Bt, Dm, Cm), Bt.nnz, "Gnnz_s",
                alg)
        if parity:
            got = sp.mttkrp(Bt, Dm, Cm)
            got = got.todense_device() if hasattr(got, "todense_device") else torch.as_tensor(np.asarray(got)).to(DEV)
            co, dv = Bt._dev()
            contrib = dv.double()[:, None] * Dm[co[2]].double() * Cm[co[1]].double()
            wantm = torch.zeros((I_, J), dtype=torch.float64, device=DEV).index_add_(0, co[0], contrib)
            r["parity"] = {"vs": "fp64 restatement sum_kl B[i,k,l] D[l,j] C[k,j], rtol 2e-5",
                           "values_close": bool(torch.allclose(got.double(), wantm, rtol=2e-5, atol=1e-9))}
            del contrib, wantm

    if "mttkrp_mode" in which:
        # K9's config, mode 0, next to the fused mttkrp above (same seeds)
        I_, K_, L_, J = 10_000, 10_000, 1_000, 32
        Bt = rand_coo((I_, K_, L_), 10_000_000, 31, torch.float32)
        g = torch.Generator(device=DEV).manual_seed(32)
        Dm = torch.rand((L_, J), generator=g, device=DEV, dtype=torch.float32)
        Cm = torch.rand((K_, J), generator=g, device=DEV, dtype=torch.float32)
        alg = Bt.nnz * (3 * 4 + 4) + Bt.nnz * 2 * J * 4 + I_ * J * 4
        r = rec("MTTKRP mttkrp_mode mode 0 (1e4 x 1e4 x 1e3, nnz 1e7, J=32 f32)",
                lambda: sp.mttkrp_mode(Bt, [None, Cm, Dm], 0), Bt.nnz, "Gnnz_s", alg)
        if parity:
            got = sp.mttkrp_mode(Bt, [None, Cm, Dm], 0)
            co, dv = Bt._dev()
            contrib = dv.double()[:, None] * Cm[co[1]].double() * Dm[co[2]].double()
            wantm = torch.zeros((I_, J), dtype=torch.float64, device=DEV).index_add_(0, co[0], contrib)
            r["parity"] = {"vs": "fp64 restatement sum_kl B[i,k,l] C[k,j] D[l,j], rtol 2e-5",
                           "values_close": bool(torch.allclose(got.double(), wantm, rtol=2e-5, atol=0))}
            del contrib, wantm
        del Bt, Dm, Cm
        res.update(_mttkrp_mode_order3(rec, parity))
    if "masked" in which:
        res.update(_masked(rec, parity))
    if "ttmc" in which:
        res.update(_ttmc(rec, parity))
    if "tttp" in which:
        res.update(_tttp(rec, parity))
    if "ttm" in which:
        res.update(_ttm(rec, parity))
    if "completion" in which:
        res.update(_completion(rec, parity))
    if "cp_apr" in which:
        res.update(_cp_apr(rec, parity))
    if "sptc" in which:
        res.update(_sptc(rec, parity))
    torch.cuda.empty_cache()
    return res


def _card():
    """Name and power limit of the GPU, read next to the timings."""
    import subprocess

    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader",
                        "-i", str(DEV.index or 0)], capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(DEV)


def _graph_from_edges(n, i, j):
    """Symmetric 0/1 float32 adjacency matrix (COO) of the edges (i, j), without self-loops or duplicates."""
    keep = i != j
    i, j = i[keep], j[keep]
    keys = torch.unique(torch.cat([i * n + j, j * n + i]))
    coords = torch.stack([torch.div(keys, n, rounding_mode="floor"), keys % n])
    return sp.COO(coords, torch.ones(keys.numel(), device=DEV, dtype=torch.float32), shape=(n, n),
                  has_duplicates=False, sorted=True)


def _rmat_edges(n_log2, m, seed, probs=(0.57, 0.19, 0.19, 0.05)):
    g = torch.Generator(device=DEV).manual_seed(seed)
    i = torch.zeros(m, dtype=torch.int64, device=DEV)
    j = torch.zeros(m, dtype=torch.int64, device=DEV)
    cut = torch.tensor(np.cumsum(probs)[:3], device=DEV, dtype=torch.float32)
    for _ in range(n_log2):
        q = torch.bucketize(torch.rand(m, generator=g, device=DEV), cut)
        i = i * 2 + (q >= 2).to(torch.int64)
        j = j * 2 + (q % 2).to(torch.int64)
    return i, j


def _masked(rec, parity):
    """Masked SpGEMM on graphs (mask = a = b = the adjacency matrix A, f32): masked_matmul(A, A, A) against the
    unfused A * (A @ A).  Byte model per call (from the degrees d_i of A, with nnz = sum d_i):
      mask stream    nnz * (4 index + 4 value + 4 result) + indptr
      A staging      nnz * (4 + 4): every row of A is staged once per chunk that touches its mask row
      B^T indices    sum over mask entries (i, j) of d_j * 4 = sum_j d_j^2 * 4 (plus 8 B of extent per entry)
      value gathers  4 B per match; a match of entry (i, j) is a triangle through the edge, 6 per triangle
    Unfused memory: K4's upper-bound layout holds min(P_i, n) (index + value) slots per row (P_i = sum of the
    degrees of the row's neighbours) and its result (int64 index + value) per product, then the multiply merges the
    whole product with the mask.  The unfused call is run in row blocks to keep the footprint moderate: rows of
    A * (A @ A) depend only on the same rows of the mask and of A, so the values are those of one call."""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import _mock_masked as MM

    out = {}
    card = _card()
    n_log2 = 20
    n = 1 << n_log2
    m = n * 16
    g = torch.Generator(device=DEV).manual_seed(51)
    uniform = _graph_from_edges(n, torch.randint(0, n, (m,), generator=g, device=DEV),
                                torch.randint(0, n, (m,), generator=g, device=DEV))
    rmat = _graph_from_edges(n, *_rmat_edges(n_log2, m, 52))
    for gname, A in (("uniform", uniform), ("R-MAT", rmat)):
        A._dev()
        keys = A.sorted_keys()
        deg = torch.bincount(torch.div(keys, n, rounding_mode="floor"), minlength=n).to(torch.float64)
        nnz = A.nnz
        products = float((deg * deg).sum())  # sum_k |A_:,k| |A_k,:| for symmetric A
        res = sp.masked_matmul(A, A, A)
        matches = float(res._data_dev().double().sum())
        alg = nnz * 12 + (n + 1) * 4 + nnz * 8 + products * 4 + nnz * 8 + matches * 4
        p_row = torch.zeros(n, dtype=torch.float64, device=DEV).index_add_(
            0, torch.div(keys, n, rounding_mode="floor"), deg[keys % n])
        unfused_bytes = float(torch.clamp(p_row, max=n).sum()) * 8 + products * 12 + nnz * 16
        name = f"masked_matmul {gname} graph 2^20 vertices, avg degree {nnz / n:.1f}, f32"
        r = rec(name, lambda: sp.masked_matmul(A, A, A), nnz, "G_mask_entries_s", alg, reps=5)
        r.update({"card": card, "mask_nnz": int(nnz), "products_unfused": int(products), "byte_model": int(alg),
                  "unfused_memory_model_bytes": int(unfused_bytes), "triangles_fused": matches / 6,
                  "max_degree": int(deg.max())})
        if gname == "uniform":
            blocks = 4
            step = n // blocks
            parts = [A[r0:r0 + step] for r0 in range(0, n, step)]
            for p in parts:
                p._dev()

            def unfused():
                return [p * (p @ A) for p in parts]

            best, med = timeit(unfused, reps=3, warm=1)
            ref = unfused()
            rk = torch.cat([x.sorted_keys() + b * step * n for b, x in enumerate(ref)])
            rv = torch.cat([x._data_dev() for x in ref])
            inm = torch.isin(rk, keys)
            fk, fv = res.sorted_keys(), res._data_dev()
            r["unfused"] = {"ms_best": round(best, 4), "ms_median": round(med, 4), "row_blocks": blocks,
                            "card": _card(), "triangles": float(rv.double().sum()) / 6,
                            "entries_outside_mask": int((~inm).sum())}
            r["parity"] = {"vs": "unfused A * (A @ A) of the package, restricted to the mask",
                           "fused_equals_unfused_on_mask_bitwise": bool(
                               torch.equal(rk[inm], fk) and torch.equal(rv[inm].view(torch.int32),
                                                                           fv.view(torch.int32))),
                           "triangles_equal": r["unfused"]["triangles"] == matches / 6}
            r["speedup_vs_unfused"] = round(med / r["ms_median"], 2)
            del ref, rk, rv, inm, parts
        elif parity:
            # six random rows and one long row (the degree nearest 512; the hubs take minutes in the CPU restatement)
            rows = np.random.default_rng(53).choice(n, 6, replace=False).tolist() + [int((deg - 512).abs().argmin())]
            mv, mi, mp = (x.cpu().numpy() for x in A.asformat("gcxs", compressed_axes=(0,))._dev())
            full = torch.zeros(nnz, dtype=torch.float32, device=DEV)
            full[torch.searchsorted(keys, res.sorted_keys())] = res._data_dev()
            fullh = full.cpu().numpy()
            ok = True
            for i in rows:
                pos, want = MM.order_contract(mp, mi, mv, mp, mi, mv, mp, mi, mv, rows=[i])
                ok &= bool(np.array_equal(fullh[pos].view(np.uint32), want.view(np.uint32)))
            r["parity"] = {"vs": "CPU restatement of the order (tests/_mock_masked.py) on 7 sampled rows",
                           "sampled_rows_bit_exact": ok}
        out[name] = r
        del res, keys, deg, p_row
    return out


def _mttkrp_mode_order3(rec, parity):
    """CP-ALS workload: (1e6, 1e6, 100) with 1e8 uniform entries, R = 32, f32, factors on the device.  Modes 0 and 1
    have ~100 entries per slice, mode 2 has 100 slices of ~1e6 entries (the skewed case)."""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import _tensor_order as TO

    shape, R = (1_000_000, 1_000_000, 100), 32
    X = rand_coo(shape, 100_000_000, 41, torch.float32)
    g = torch.Generator(device=DEV).manual_seed(42)
    U = [torch.rand((s, R), generator=g, device=DEV, dtype=torch.float32) for s in shape]
    coords, vals = X._dev()
    nnz, N, ib, vb = X.nnz, 3, 4, 4
    ch = sp._kernels.mttkrp_mode_chunk()
    out = {}
    for mode in range(N):
        X._mode_streams = None  # first call: builds the mode stream (sort + gathers + narrowing)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        sp.mttkrp_mode(X, U, mode)
        torch.cuda.synchronize()
        first = (time.perf_counter() - t0) * 1e3
        alg = nnz * (N * ib + vb) + nnz * (N - 1) * R * vb + shape[mode] * R * vb
        name = f"mttkrp_mode order-3 (1e6,1e6,100) nnz 1e8 R=32 f32 mode {mode}"
        r = rec(name, lambda: sp.mttkrp_mode(X, U, mode), nnz, "Gnnz_s", alg)
        r["first_call_ms"] = round(first, 3)
        r["gather_model_bytes"] = int(alg)
        if parity:
            got = sp.mttkrp_mode(X, U, mode)
            want = torch.zeros((shape[mode], R), dtype=torch.float64, device=DEV)
            for s in range(0, nnz, 10_000_000):
                c = coords[:, s:s + 10_000_000]
                p = vals[s:s + 10_000_000].double()[:, None]
                for m in range(N):
                    if m != mode:
                        p = p * U[m][c[m]].double()
                want.index_add_(0, c[mode], p)
            close = bool(torch.allclose(got.double(), want, rtol=2e-5, atol=0))
            del want
            rows = np.random.default_rng(mode).choice(shape[mode], 4, replace=False)
            exact = TO.sampled_rows_exact(got, coords, vals, U, mode, rows, ch, kron=False)
            r["parity"] = {"vs": "fp64 device restatement (all rows, rtol 2e-5) + 4 sampled rows bit-compared with "
                                 "the CPU restatement of the order (tests/_tensor_order.py)",
                           "values_close": close, "sampled_rows_bit_exact": exact}
        out[name] = r
    del X, U, coords, vals
    return out


def _ttmc_parity(X, U, mode, got, ranks, sample_rows, seed):
    """fp64 device restatement of every row (one block of R_last columns per leading digit, entries in blocks of 1e7)
    and `sample_rows` rows bit-compared with the CPU restatement of the order (tests/_tensor_order.py)."""
    import _tensor_order as TO

    coords, vals = X._dev()
    shape, nnz = X.shape, X.nnz
    a, b = [m for m in range(3) if m != mode]
    Rb = ranks[b]
    close = True
    for ra in range(ranks[a]):
        want = torch.zeros((shape[mode], Rb), dtype=torch.float64, device=DEV)
        for s in range(0, nnz, 10_000_000):
            c = coords[:, s:s + 10_000_000]
            p = vals[s:s + 10_000_000].double() * U[a][c[a], ra].double()
            want.index_add_(0, c[mode], p[:, None] * U[b][c[b]].double())
        close &= bool(torch.allclose(got[:, ra * Rb:(ra + 1) * Rb].double(), want, rtol=2e-5, atol=0))
        del want
    rows = np.random.default_rng(seed).choice(shape[mode], sample_rows, replace=False)
    exact = TO.sampled_rows_exact(got, coords, vals, U, mode, rows, sp._kernels.mttkrp_mode_chunk(), kron=True)
    return {"vs": f"fp64 device restatement (all rows, rtol 2e-5) + {sample_rows} sampled rows bit-compared with the "
                  "CPU restatement of the order (tests/_tensor_order.py)",
            "values_close": close, "sampled_rows_bit_exact": exact}


def _ttmc_models(X, ranks, mode, vb=4, ib=4):
    """Byte and op models of one ttmc_mode call from shapes (f32, int32 stream).  Bytes: the stream (N coordinates +
    value) once per column tile; one full row of every other factor per entry (every gather from HBM: an upper bound,
    the rows are largely L2 hits); the output; the pieces (written and read back by the combine kernel).  Ops: one
    multiply and one add per entry and column, plus the prefix multiplies (one per leading mode, per entry and lane)."""
    N, nnz = X.ndim, X.nnz
    others = [m for m in range(N) if m != mode]
    W = int(np.prod([ranks[m] for m in others]))
    vec = 16 // vb
    packs = -(-W // vec)
    G = 16 if packs > 8 else 8 if packs > 4 else 4 if packs > 2 else 2 if packs > 1 else 1  # dispatch_ttmc's groups
    tiles = -(-W // (G * vec))
    nchunks = -(-nnz // 512)
    stream = tiles * nnz * (N * ib + vb)
    gathers = nnz * sum(ranks[m] for m in others) * vb
    output = X.shape[mode] * W * vb
    pieces = 2 * 2 * nchunks * (-(-W // 4) * 4) * vb
    total = stream + gathers + output + pieces
    ops = nnz * (2 * W + (len(others) - 1) * packs)
    sm_ops = 132 * 128 * 1.98e9  # FP32 lanes x the H100 SXM boost clock: separate multiplies and adds per second
    return {"W": W, "column_tiles": tiles, "bytes": {"stream": stream, "factor_gathers": gathers, "output": output,
                                                     "pieces": pieces, "total": total},
            "op_model": ops, "model_ms_bytes_at_3.35TBs": round(total / 3.35e12 * 1e3, 3),
            "model_ms_ops_at_3.3e13": round(ops / sm_ops * 1e3, 3)}


def _ttmc(rec, parity):
    """Tucker / HOOI step: ttmc_mode on the CP-ALS workload of mttkrp_mode ((1e6, 1e6, 100), nnz 1e8, f32) at R_m = 16
    (W = 256, every mode) and R_m = 32 (W = 1024, mode 0), and on K9's config at R_m = 8 (W = 64) next to the unfused
    einsum("ijk,jb,kc->ibc"), whose nnz * W broadcast products are what the fused kernel avoids."""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    out = {}
    card = _card()
    shape = (1_000_000, 1_000_000, 100)
    X = rand_coo(shape, 100_000_000, 61, torch.float32)
    g = torch.Generator(device=DEV).manual_seed(62)
    for R, modes in ((16, (0, 1, 2)), (32, (0,))):
        U = [torch.rand((s, R), generator=g, device=DEV, dtype=torch.float32) for s in shape]
        for mode in modes:
            X._mode_streams = None  # first call: builds the mode stream (sort + gathers + narrowing)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            sp.ttmc_mode(X, U, mode)
            torch.cuda.synchronize()
            first = (time.perf_counter() - t0) * 1e3
            models = _ttmc_models(X, [R] * 3, mode)
            name = f"ttmc_mode order-3 (1e6,1e6,100) nnz 1e8 R_m={R} (W={R * R}) f32 mode {mode}"
            r = rec(name, lambda: sp.ttmc_mode(X, U, mode), X.nnz, "Gnnz_s", models["bytes"]["total"])
            r.update({"card": card, "first_call_ms": round(first, 3), **models})
            if parity:
                got = sp.ttmc_mode(X, U, mode)
                r["parity"] = _ttmc_parity(X, U, mode, got, [R] * 3, 4, 70 + mode)
                del got
            out[name] = r
            torch.cuda.empty_cache()
        del U
    del X
    torch.cuda.empty_cache()

    I_, K_, L_, R = 10_000, 10_000, 1_000, 8
    Bt = rand_coo((I_, K_, L_), 10_000_000, 31, torch.float32)
    g = torch.Generator(device=DEV).manual_seed(63)
    U = [None] + [torch.rand((s, R), generator=g, device=DEV, dtype=torch.float32) for s in (K_, L_)]
    models = _ttmc_models(Bt, [R] * 3, 0)
    name = "ttmc_mode K9 config (1e4 x 1e4 x 1e3, nnz 1e7) R_m=8 (W=64) f32 mode 0"
    r = rec(name, lambda: sp.ttmc_mode(Bt, U, 0), Bt.nnz, "Gnnz_s", models["bytes"]["total"])
    r.update({"card": card, **models})
    got = sp.ttmc_mode(Bt, U, 0)
    if parity:
        r["parity"] = _ttmc_parity(Bt, U, 0, got, [R] * 3, 4, 73)
    Uh = [u.cpu().numpy() for u in U[1:]]
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats(DEV)
    base = torch.cuda.memory_allocated(DEV)
    unf = {"expression": 'einsum("ijk,jb,kc->ibc", X, U1, U2)', "card": _card()}
    try:
        t0 = time.perf_counter()
        ref = sp.einsum("ijk,jb,kc->ibc", Bt, *Uh)
        dense = ref.todense_device() if hasattr(ref, "todense_device") else torch.as_tensor(np.asarray(ref)).to(DEV)
        torch.cuda.synchronize()
        unf["ms_first"] = round((time.perf_counter() - t0) * 1e3, 3)
        del ref
        best, med = timeit(lambda: sp.einsum("ijk,jb,kc->ibc", Bt, *Uh), reps=3, warm=1)
        unf.update({"ms_best": round(best, 4), "ms_median": round(med, 4), "fits": True,
                    "peak_extra_bytes": int(torch.cuda.max_memory_allocated(DEV) - base),
                    "values_close_to_fused": bool(torch.allclose(dense.reshape(I_, R * R), got, rtol=2e-5, atol=1e-6))})
        r["speedup_vs_unfused"] = round(med / r["ms_median"], 2)
        del dense
    except (torch.OutOfMemoryError, RuntimeError) as e:  # the broadcast products do not fit on the card
        unf.update({"fits": False, "error": str(e).splitlines()[0][:200],
                    "peak_extra_bytes_before_failure": int(torch.cuda.max_memory_allocated(DEV) - base)})
    r["unfused"] = unf
    out[name] = r
    del Bt, U, got
    torch.cuda.empty_cache()
    return out


def _tttp_parity(X, U, got, samples, seed):
    """Every entry against an fp64 device restatement (rtol 2e-5) and `samples` sampled entries bit-compared with the
    CPU restatement of the order (tests/_tensor_order.py).  X is COO; `got` has X's pattern (nothing pruned)."""
    import _tensor_order as TO

    coords, vals = X._dev()
    gv = got._data_dev()
    close = got.nnz == X.nnz
    for s in range(0, X.nnz, 10_000_000):
        c = coords[:, s:s + 10_000_000]
        m = U[0][c[0]].double()
        for k in range(1, X.ndim):
            m = m * U[k][c[k]].double()
        close &= bool(torch.allclose(gv[s:s + 10_000_000].double(), vals[s:s + 10_000_000].double() * m.sum(1),
                                     rtol=2e-5, atol=0))
        del m
    pick = torch.from_numpy(np.sort(np.random.default_rng(seed).choice(X.nnz, samples, replace=False))).to(DEV)
    want = TO.values(coords[:, pick].cpu().numpy(), vals[pick].cpu().numpy(), [u.cpu().numpy() for u in U],
                     np.float32)
    return {"vs": f"fp64 device restatement (all entries, rtol 2e-5) + {samples} sampled entries bit-compared with the "
                  "CPU restatement of the order (tests/_tensor_order.py)",
            "values_close": close, "sampled_entries_bit_exact": TO.same_bits(gv[pick].cpu().numpy(), want)}


def _tttp_models(X, R, vb=4, ib=4):
    """Byte model of one tttp call from shapes (f32, int32 coordinates): the entry stream, the output values, and one
    R-column row of every factor per entry counted as if every gather came from HBM (most are L2 hits, so the kernel
    may beat this model; it is not an HBM share)."""
    N, nnz = X.ndim, X.nnz
    b = {"stream": nnz * (N * ib + vb), "output": nnz * vb, "factor_gathers": nnz * N * R * vb}
    b["total"] = sum(b.values())
    return {"bytes": b, "model_ms_bytes_at_3.35TBs": round(b["total"] / 3.35e12 * 1e3, 3)}


def _no_zero_values(X):
    """X with 0.1 added to every value: tttp of a positive model then prunes nothing, so results align with X."""
    coords, vals = X._dev()
    return sp.COO(coords, vals + 0.1, shape=X.shape, has_duplicates=False, sorted=True)


def _tttp(rec, parity):
    """CP model at the stored entries: tttp on the CP-ALS workload of mttkrp_mode ((1e6, 1e6, 100), nnz 1e8, R = 32,
    f32, COO and one GCXS layout); at order 2 on C4's shape next to sddmm, alternating; and on K9's config next to the
    unfused einsum("ijk,ir,jr,kr->ijk"), whose nnz * R products are what the fused kernel avoids."""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import _tensor_order as TO

    out = {}
    card = _card()
    shape, R = (1_000_000, 1_000_000, 100), 32
    X = _no_zero_values(rand_coo(shape, 100_000_000, 81, torch.float32))
    g = torch.Generator(device=DEV).manual_seed(82)
    U = [torch.rand((s, R), generator=g, device=DEV, dtype=torch.float32) + 0.05 for s in shape]
    models = _tttp_models(X, R)
    name = "tttp order-3 (1e6,1e6,100) nnz 1e8 R=32 f32 COO"
    r = rec(name, lambda: sp.tttp(X, U), X.nnz, "Gnnz_s", models["bytes"]["total"])
    r.update({"card": card, **models})
    if parity:
        got = sp.tttp(X, U)
        r["parity"] = _tttp_parity(X, U, got, 10_000, 83)
        del got
    out[name] = r
    G = X.asformat("gcxs", compressed_axes=(2,))
    name = "tttp order-3 (1e6,1e6,100) nnz 1e8 R=32 f32 GCXS compressed_axes=(2,)"
    r = rec(name, lambda: sp.tttp(G, U), X.nnz, "Gnnz_s")
    r["card"] = card
    if parity:
        gc = sp.tttp(G, U).tocoo()
        r["parity"] = {"vs": "the COO result (GCXS result converted to COO)",
                       "bit_exact": bool(TO.same_bits(gc.data, sp.tttp(X, U).data))}
        del gc
    out[name] = r
    del X, G, U
    torch.cuda.empty_cache()

    # order 2 at C4's shape: tttp against sddmm on the same inputs, alternating
    M = N = 1_000_000
    K = 256
    S = _no_zero_values(rand_coo((M, N), 100_000_000, 84, torch.float32))
    g = torch.Generator(device=DEV).manual_seed(85)
    A, Bt = (torch.rand((n, K), generator=g, device=DEV, dtype=torch.float32) for n in (M, N))
    t_fns = {"tttp": lambda: sp.tttp(S, [A, Bt]), "sddmm": lambda: sp.sddmm(S, A, Bt, b_transposed=True)}
    times = {k: [] for k in t_fns}
    for k, fn in t_fns.items():
        fn()
    for _ in range(5):
        for k, fn in t_fns.items():
            times[k].append(timeit(fn, reps=1, warm=0)[0])
    a, b = sp.tttp(S, [A, Bt]), sp.sddmm(S, A, Bt, b_transposed=True)
    models = _tttp_models(S, K)
    name = "tttp order-2 C4 shape (1e6^2, nnz 1e8) R=K=256 f32 vs sddmm"
    r = {"ms_median": round(float(np.median(times["tttp"])), 4), "ms_best": round(min(times["tttp"]), 4),
         "sddmm_ms_median": round(float(np.median(times["sddmm"])), 4), "sddmm_ms_best": round(min(times["sddmm"]), 4),
         "card": card, **models,
         "values_close_to_sddmm": bool(a.nnz == b.nnz and torch.allclose(a._data_dev(), b._data_dev(), rtol=2e-5))}
    if parity:
        r["parity"] = _tttp_parity(S, [A, Bt], a, 10_000, 86)
    print(name, r, flush=True)
    out[name] = r
    del S, A, Bt, a, b
    torch.cuda.empty_cache()

    # K9's config: tttp against the unfused expression
    Bk = _no_zero_values(rand_coo((10_000, 10_000, 1_000), 10_000_000, 31, torch.float32))
    g = torch.Generator(device=DEV).manual_seed(87)
    U = [torch.rand((s, R), generator=g, device=DEV, dtype=torch.float32) + 0.05 for s in Bk.shape]
    models = _tttp_models(Bk, R)
    name = "tttp K9 config (1e4 x 1e4 x 1e3, nnz 1e7) R=32 f32"
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats(DEV)
    base = torch.cuda.memory_allocated(DEV)
    r = rec(name, lambda: sp.tttp(Bk, U), Bk.nnz, "Gnnz_s", models["bytes"]["total"])
    r.update({"card": card, "peak_extra_bytes": int(torch.cuda.max_memory_allocated(DEV) - base), **models})
    got = sp.tttp(Bk, U)
    if parity:
        r["parity"] = _tttp_parity(Bk, U, got, 10_000, 88)
    Uh = [u.cpu().numpy() for u in U]
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats(DEV)
    base = torch.cuda.memory_allocated(DEV)
    unf = {"expression": 'einsum("ijk,ir,jr,kr->ijk", X, U0, U1, U2)', "card": _card()}
    try:
        ref = sp.einsum("ijk,ir,jr,kr->ijk", Bk, *Uh)
        best, med = timeit(lambda: sp.einsum("ijk,ir,jr,kr->ijk", Bk, *Uh), reps=3, warm=1)
        ref = ref.asformat("coo")
        unf.update({"ms_best": round(best, 4), "ms_median": round(med, 4), "fits": True,
                    "peak_extra_bytes": int(torch.cuda.max_memory_allocated(DEV) - base),
                    "values_close_to_fused": bool(ref.nnz == got.nnz and np.array_equal(ref.coords, got.coords)
                                                  and np.allclose(ref.data, got.data, rtol=2e-5, atol=0))})
        r["speedup_vs_unfused"] = round(med / r["ms_median"], 2)
        del ref
    except (torch.OutOfMemoryError, RuntimeError) as e:  # the broadcast products do not fit on the card
        unf.update({"fits": False, "error": str(e).splitlines()[0][:200],
                    "peak_extra_bytes_before_failure": int(torch.cuda.max_memory_allocated(DEV) - base)})
    r["unfused"] = unf
    out[name] = r
    del Bk, U, got
    torch.cuda.empty_cache()
    return out


def _ttm_models(X, nf, R, vb=4, ib=4):
    """Byte model of one ttm_mode call with the fiber stream cached (f32, int32 indices): the stream (entries, and per
    fiber its pointer, group, key and P key), one R-column row of U per entry counted as if every gather came from HBM
    (most are L2 hits), the n_fibers * R slots (value, key, flag) and the scan over the flags (read, positions)."""
    nnz = X.nnz
    b = {"stream": nnz * (ib + vb) + nf * (2 * ib + 16), "u_gathers": nnz * R * vb, "slots": nf * R * (vb + 9),
         "scan": nf * R * 9}
    b["total"] = sum(b.values())
    return {"bytes": b, "model_ms_bytes_at_3.35TBs": round(b["total"] / 3.35e12 * 1e3, 3)}


def _ttm_parity(X, U, mode, got, samples, seed):
    """Every value against an fp64 device restatement (per-fiber index_add of v * U[k], rtol 2e-5), and `samples`
    sampled fibers bit-compared with the CPU restatement of the order (tests/_tensor_order.py)."""
    import _tensor_order as TO

    coords, vals = X._dev()
    shape, N = X.shape, X.ndim
    others = [m for m in range(N) if m != mode]

    def fiber_keys(c):
        k = torch.zeros(c.shape[1], dtype=torch.int64, device=DEV)
        for m in others:
            k = k * shape[m] + c[m].to(torch.int64)
        return k

    Ud = U.double()
    fk = fiber_keys(coords)
    uk, inv = torch.unique(fk, return_inverse=True)
    del fk
    want = torch.zeros((uk.numel(), Ud.shape[1]), dtype=torch.float64, device=DEV)
    mag = torch.zeros_like(want)  # sum of |v * U| per (fiber, r): the scale of the f32 rounding error
    step = 20_000_000
    for s in range(0, X.nnz, step):
        prod = vals[s:s + step].double()[:, None] * Ud[coords[mode, s:s + step]]
        want.index_add_(0, inv[s:s + step], prod)
        mag.index_add_(0, inv[s:s + step], prod.abs())
        del prod
    # a serial sum of L rounded f32 products is within (L + 1) * 2**-24 * sum |v * U| of the exact one (the standard
    # recursive-summation bound); long fibers can exceed a plain rtol, so each value gets the larger of the two
    flen = torch.bincount(inv, minlength=uk.numel()).double()
    del inv
    R = Ud.shape[1]
    q_ext = int(np.prod(shape[mode + 1:], dtype=np.int64))
    keys, gv = got.sorted_keys(), got._data_dev()
    close, gfk_parts = True, []
    for s in range(0, got.nnz, step):
        k = keys[s:s + step]
        r = torch.div(k, q_ext, rounding_mode="floor") % R
        gfk = torch.div(k, q_ext * R, rounding_mode="floor") * q_ext + k % q_ext
        gfk_parts.append(gfk)
        fi = torch.searchsorted(uk, gfk)
        w = want[fi, r]
        tol = torch.maximum(2e-5 * w.abs(), (flen[fi] + 1) * 2.0**-24 * mag[fi, r])
        close &= bool(((gv[s:s + step].double() - w).abs() <= tol).all())
    del want, mag, flen
    pick = torch.from_numpy(np.sort(np.random.default_rng(seed).choice(uk.numel(), samples, replace=False))).to(DEV)
    chosen = uk[pick]
    sel = torch.isin(fiber_keys(coords), chosen)
    gsel = torch.isin(torch.cat(gfk_parts), chosen)
    rc, rv = TO.result(coords[:, sel].cpu().numpy(), vals[sel].cpu().numpy(), shape, U.cpu().numpy(), mode,
                       np.float32)
    got_c = torch.stack(torch.unravel_index(keys[gsel], got.shape)).cpu().numpy()
    exact = bool(np.array_equal(got_c, rc) and TO.same_bits(gv[gsel].cpu().numpy(), rv))
    return {"vs": f"fp64 device restatement (all values, within max(rtol 2e-5, (L + 1) * 2**-24 * sum |v * U|) for a "
                  f"fiber of L entries) + {samples} sampled fibers bit-compared with the CPU restatement of the order "
                  "(tests/_tensor_order.py)",
            "values_close": close, "sampled_fibers_bit_exact": exact}


def _ttm_vs_tensordot(name, X, mode, R, seed, card, parity):
    """ttm_mode against moveaxis(tensordot(..., return_type=COO), -1, mode), alternating, median of 5 each, and the peak
    device memory of one call of each beyond the inputs; ttm_mode's first call is measured, so its peak includes
    building the fiber stream that then stays cached on X."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    U = torch.rand((X.shape[mode], R), generator=g, device=DEV, dtype=torch.float32)
    fns = {"ttm_mode": lambda: sp.ttm_mode(X, U, mode),
           "tensordot": lambda: sp.moveaxis(sp.tensordot(X, U, axes=([mode], [0]), return_type=sp.COO), -1, mode)}
    peak = {}
    for k, fn in fns.items():
        X._mode_streams = None
        fn()  # warms the kernels; for tensordot, also the first call's allocations
        X._mode_streams = None
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats(DEV)
        base = torch.cuda.memory_allocated(DEV)
        fn()
        torch.cuda.synchronize()
        peak[k] = int(torch.cuda.max_memory_allocated(DEV) - base)
    times = {k: [] for k in fns}
    for _ in range(5):
        for k, fn in fns.items():
            times[k].append(timeit(fn, reps=1, warm=0)[0])
    got, want = fns["ttm_mode"](), fns["tensordot"]()
    nf = int(X._mode_streams[("fiber", mode, True)][5].numel())
    r = {"ms_median": round(float(np.median(times["ttm_mode"])), 4), "ms_best": round(min(times["ttm_mode"]), 4),
         "tensordot_ms_median": round(float(np.median(times["tensordot"])), 4),
         "tensordot_ms_best": round(min(times["tensordot"]), 4),
         "speedup_vs_tensordot": round(float(np.median(times["tensordot"]) / np.median(times["ttm_mode"])), 2),
         "peak_extra_bytes_incl_fiber_stream": peak["ttm_mode"], "tensordot_peak_extra_bytes": peak["tensordot"],
         "card": card, "n_fibers": nf, **_ttm_models(X, nf, R)}
    if parity:
        gb, wb = got._data_dev(), want._data_dev()
        r["parity"] = _ttm_parity(X, U, mode, got, 2_000, seed + 1)
        r["parity"]["whole_result_bit_exact_vs_tensordot"] = bool(
            got.nnz == want.nnz and torch.equal(got.sorted_keys(), want.sorted_keys())
            and torch.equal(gb.view(torch.int32), wb.view(torch.int32)))
    print(name, r, flush=True)
    return r


def _ttm(rec, parity):
    """Mode-n TTM with a sparse result: short fibers (about one entry each, the output-write bound regime) at modes 0
    and 2, long fibers (about 100 entries, U gathers mostly L2 hits), and two shapes where tensordot still fits -- one
    uniform, one with Zipf fiber lengths up to 1e6 entries -- timed against it alternating, with both calls' peak extra
    device memory."""
    sys.path.insert(0, os.path.join(ROOT, "tests"))

    out = {}
    card = _card()
    cases = (("short fibers (1e6,1e6,100) nnz 1e8", (1_000_000, 1_000_000, 100), (0, 2), 8, 91),
             ("long fibers (1e3,1e3,1e5) nnz 1e8", (1_000, 1_000, 100_000), (2,), 64, 93))
    for label, shape, modes, R, seed in cases:
        X = rand_coo(shape, 100_000_000, seed, torch.float32)
        g = torch.Generator(device=DEV).manual_seed(seed + 1)
        for mode in modes:
            U = torch.rand((shape[mode], R), generator=g, device=DEV, dtype=torch.float32)
            torch.cuda.synchronize()
            X._mode_streams = None
            t0 = time.perf_counter()
            got = sp.ttm_mode(X, U, mode)
            torch.cuda.synchronize()
            first = (time.perf_counter() - t0) * 1e3
            nf = int(X._mode_streams[("fiber", mode, True)][5].numel())
            models = _ttm_models(X, nf, R)
            name = f"ttm_mode {label} mode {mode} R={R} f32"
            r = rec(name, lambda: sp.ttm_mode(X, U, mode), X.nnz, "Gnnz_s", models["bytes"]["total"])
            r.update({"card": card, "first_call_ms_incl_fiber_stream": round(first, 3), "n_fibers": nf,
                      "out_nnz": got.nnz, **models})
            if parity:
                r["parity"] = _ttm_parity(X, U, mode, got, 2_000, seed + 2)
            out[name] = r
            del got, U
            X._mode_streams = None
            torch.cuda.empty_cache()
        del X
        torch.cuda.empty_cache()

    # tensordot still fits: fused against unfused, alternating, with the peak extra memory of each
    shape, mode, R = (10_000, 1_000, 1_000), 2, 16
    X = rand_coo(shape, 10_000_000, 95, torch.float32)
    name = "ttm_mode (1e4,1e3,1e3) nnz 1e7 mode 2 R=16 f32 vs tensordot(return_type=COO)"
    out[name] = _ttm_vs_tensordot(name, X, mode, R, 96, card, parity)
    del X
    torch.cuda.empty_cache()

    # skewed fiber lengths (Zipf, the longest 1e6 entries) where tensordot still fits
    shape, mode, R = (10_000, 1_000, 2_000_000), 2, 8
    g = torch.Generator(device=DEV).manual_seed(98)
    size = int(np.prod(shape))
    parts = [torch.randint(0, size, (20_000_000,), generator=g, device=DEV)]
    fibers = torch.randint(0, shape[0] * shape[1], (4_000,), generator=g, device=DEV).tolist()
    for i, fib in enumerate(fibers, start=1):
        n = int(1e6 * i ** -1.2)
        if n < 64:
            break
        parts.append(fib * shape[2] + torch.randint(0, shape[2], (n,), generator=g, device=DEV))
    lin = torch.cat(parts)
    del parts
    X = sp.COO(torch.stack(torch.unravel_index(lin, shape)), torch.rand(lin.numel(), generator=g, device=DEV),
               shape=shape)  # duplicates summed, sorted
    del lin
    name = "ttm_mode skewed fibers (1e4,1e3,2e6) nnz 2.6e7 Zipf lengths up to 1e6, mode 2 R=8 f32 vs tensordot"
    r = _ttm_vs_tensordot(name, X, mode, R, 99, card, parity)
    fp = X._mode_streams[("fiber", mode, True)][2].to(torch.int64)
    lens = fp[1:] - fp[:-1]
    r.update({"nnz": X.nnz, "longest_fiber": int(lens.max()), "fibers_over_512": int((lens > 512).sum()),
              "entries_in_fibers_over_512": int(lens[lens > 512].sum())})
    out[name] = r
    del X, fp, lens
    torch.cuda.empty_cache()
    return out


def _completion_models(X, mode, R, vb=4, ib=4):
    """Models of one cp_completion_mode call (f32, int32 coordinates).  Bytes: the mode stream, one R-column row of
    every other factor per entry counted as if every gather came from HBM (K10's model), the result, and the crossing
    rows' scratch written and read.  Operations: R(R+1)/2 multiplies and as many adds per entry, R of each for b, and
    about R^3 / 3 per row for the factorisation and the solves, against 132 SMs x 128 FP32 lanes x 1.98 GHz without
    FMA (33.4 Tops/s: a multiply and an add are two instructions)."""
    N, nnz, rows = X.ndim, X.nnz, X.shape[mode]
    ns = R * (R + 1) // 2 + R
    nchunks = -(-nnz // 512)
    b = {"stream": nnz * (N * ib + vb), "factor_gathers": nnz * (N - 1) * R * vb, "output": rows * R * vb,
         "crossing_scratch": 2 * 2 * nchunks * ((ns + 3) // 4 * 4) * vb}
    b["total"] = sum(b.values())
    ops = {"entries": nnz * 2 * ns, "rows": int(rows * R ** 3 / 3 * 2)}
    ops["total"] = sum(ops.values())
    return {"bytes": b, "model_ms_bytes_at_3.35TBs": round(b["total"] / 3.35e12 * 1e3, 3), "ops": ops,
            "model_ms_ops_at_33.4Tops": round(ops["total"] / 33.4e12 * 1e3, 3)}


def _completion_parity(X, U, mode, R, reg, got, sample_rows, seed):
    """Every row against an fp64 device solve of (G_i + reg I) x = b_i (G and b summed in fp64), and `sample_rows`
    rows bit-compared with the CPU restatement of the order (tests/_tensor_order.py)."""
    import _tensor_order as TO

    coords, vals = X._dev()
    rows = X.shape[mode]
    others = [m for m in range(X.ndim) if m != mode]
    iu = torch.triu_indices(R, R, device=DEV)
    G = torch.zeros((rows, R, R), dtype=torch.float64, device=DEV)
    b = torch.zeros((rows, R), dtype=torch.float64, device=DEV)
    for s in range(0, X.nnz, 2_000_000):
        c = coords[:, s:s + 2_000_000]
        h = U[others[0]][c[others[0]]].double()
        for m in others[1:]:
            h = h * U[m][c[m]].double()
        G.index_put_((c[mode],), h[:, :, None] * h[:, None, :], accumulate=True)
        b.index_add_(0, c[mode], vals[s:s + 2_000_000].double()[:, None] * h)
        del h
    G += reg * torch.eye(R, dtype=torch.float64, device=DEV)
    want = torch.linalg.solve(G, b)
    del G, b
    err = ((got.double() - want).abs().amax(1) / want.abs().amax(1).clamp_min(1e-30))
    close = bool((err <= 1e-3).all())
    worst = float(err.max())
    del want, err
    (sc, sv) = X._mode_streams[(mode, True)]
    rowc = sc[mode]
    pick = np.sort(np.random.default_rng(seed).choice(rows, sample_rows, replace=False))
    bounds = torch.searchsorted(rowc, torch.from_numpy(np.stack([pick, pick + 1])).to(DEV).to(rowc.dtype)).cpu().numpy()
    Gu, bb = [], []
    for lo, hi in zip(bounds[0], bounds[1]):
        gathered = [U[m][sc[m][lo:hi].long()].cpu().numpy() for m in others]
        h, p = TO.products(None, gathered, np.float32), TO.products(sv[lo:hi].cpu().numpy(), gathered, np.float32)
        gu, bi = TO.row_system(h, p, int(lo), 512, np.float32)
        Gu.append(gu)
        bb.append(bi)
    want_rows = TO.solve(np.array(Gu), np.array(bb), np.float32(reg), np.float32)
    return {"vs": f"fp64 device solve of every row (max |x - x64| / max |x64| <= 1e-3) + {sample_rows} sampled rows "
                  "bit-compared with the CPU restatement of the order (tests/_tensor_order.py)",
            "values_close": close, "worst_row_rel_err": worst,
            "sampled_rows_bit_exact": TO.same_bits(got[torch.from_numpy(pick).to(DEV)].cpu().numpy(), want_rows)}


def _completion(rec, parity):
    """The ALS update of CP completion on the CP-ALS workload of mttkrp_mode ((1e6, 1e6, 100), nnz 1e8, f32), R = 16
    and 32, modes 0 and 2, the mode stream cached; and on K9's config (1e4, 1e4, 1e3, nnz 1e7, R = 32) next to the
    composed route: mttkrp_mode with Kronecker-squared factors for the (rows, R^2) Grams, mttkrp_mode for b, and a
    batched dense solve."""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    out = {}
    card = _card()
    reg = 1.0
    shape = (1_000_000, 1_000_000, 100)
    X = rand_coo(shape, 100_000_000, 91, torch.float32)
    for R in (16, 32):
        g = torch.Generator(device=DEV).manual_seed(92 + R)
        U = [torch.randn((s, R), generator=g, device=DEV, dtype=torch.float32) for s in shape]
        for mode in (0, 2):
            name = f"cp_completion_mode order-3 (1e6,1e6,100) nnz 1e8 R={R} mode {mode} f32"
            models = _completion_models(X, mode, R)
            r = rec(name, lambda: sp.cp_completion_mode(X, U, mode, reg), X.nnz, "Gnnz_s", models["bytes"]["total"])
            r.update({"card": card, **models})
            if parity:
                got = sp.cp_completion_mode(X, U, mode, reg)
                r["parity"] = _completion_parity(X, U, mode, R, reg, got, 8 if mode == 0 else 2, 93)
                del got
            out[name] = r
            print(name, r, flush=True)
        del U
    del X
    torch.cuda.empty_cache()

    I_, K_, L_, R = 10_000, 10_000, 1_000, 32
    X = rand_coo((I_, K_, L_), 10_000_000, 31, torch.float32)
    g = torch.Generator(device=DEV).manual_seed(94)
    U = [torch.randn((s, R), generator=g, device=DEV, dtype=torch.float32) for s in X.shape]
    sp.mttkrp_mode(X, U, 0)  # the mode stream, cached
    name = "cp_completion_mode K9 config (1e4,1e4,1e3) nnz 1e7 R=32 mode 0 f32"
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats(DEV)
    base = torch.cuda.memory_allocated(DEV)
    r = rec(name, lambda: sp.cp_completion_mode(X, U, 0, reg), X.nnz, "Gnnz_s")
    ns = R * (R + 1) // 2 + R
    r.update({"card": card, "peak_extra_bytes_torch": int(torch.cuda.max_memory_allocated(DEV) - base),
              "crossing_scratch_bytes": 2 * (-(-X.nnz // 512)) * ((ns + 3) // 4 * 4) * 4,
              **_completion_models(X, 0, R)})
    fused = sp.cp_completion_mode(X, U, 0, reg)
    out[name] = r

    coords, _ = X._dev()
    P = sp.COO(coords, torch.ones(X.nnz, device=DEV), shape=X.shape, has_duplicates=False, sorted=True)
    sp.mttkrp_mode(P, U, 0)  # X's pattern with ones, its mode stream cached too

    def unfused():
        Uk = [u[:, :, None] * u[:, None, :] for u in U]
        Gf = sp.mttkrp_mode(P, [None] + [u.reshape(u.shape[0], R * R) for u in Uk[1:]], 0).reshape(-1, R, R)
        bf = sp.mttkrp_mode(X, U, 0)
        return torch.linalg.solve(Gf + reg * torch.eye(R, device=DEV), bf)

    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats(DEV)
    base = torch.cuda.memory_allocated(DEV)
    name_u = "unfused: mttkrp_mode with Kronecker-squared factors + mttkrp_mode + torch.linalg.solve, same config"
    ru = rec(name_u, unfused, X.nnz, "Gnnz_s")
    ru.update({"card": card, "peak_extra_bytes_torch": int(torch.cuda.max_memory_allocated(DEV) - base)})
    x_u = unfused()
    ru["max_rel_diff_vs_fused"] = float(((x_u.double() - fused.double()).abs().amax(1)
                                         / fused.double().abs().amax(1).clamp_min(1e-30)).max())
    out[name_u] = ru
    del X, P, U, fused, x_u
    torch.cuda.empty_cache()
    return out


def _phi_models(X, mode, R, vb=4, ib=4):
    """Byte model of one cp_apr_phi_mode call (f32, int32 coordinates): the mode stream, one R-column row of every
    factor per entry counted as if every gather came from HBM, the result, and the crossing rows' scratch written and
    read."""
    N, nnz = X.ndim, X.nnz
    nchunks = -(-nnz // 512)
    b = {"stream": nnz * (N * ib + vb), "factor_gathers": nnz * N * R * vb, "output": X.shape[mode] * R * vb,
         "crossing_scratch": 2 * 2 * nchunks * ((R + 3) // 4 * 4) * vb}
    b["total"] = sum(b.values())
    return {"bytes": b, "model_ms_bytes_at_3.35TBs": round(b["total"] / 3.35e12 * 1e3, 3)}


def _alternate(fns, reps=5, warm=2):
    """Median ms of each callable, the callables timed in turn within every repetition."""
    for _ in range(warm):
        for f in fns.values():
            f()
    torch.cuda.synchronize()
    ts = {k: [] for k in fns}
    for _ in range(reps):
        for k, f in fns.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            f()
            torch.cuda.synchronize()
            ts[k].append((time.perf_counter() - t0) * 1e3)
    return {k: round(float(np.median(v)), 4) for k, v in ts.items()}


def _phi_parity(X, U, mode, eps, got, sample_rows, seed):
    """Every row against an fp64 device evaluation, and `sample_rows` rows bit-compared with the CPU restatement of
    the order (tests/_cp_apr_order.py)."""
    import _cp_apr_order as CA

    coords, vals = X._dev()
    rows, R = X.shape[mode], got.shape[1]
    want = torch.zeros((rows, R), dtype=torch.float64, device=DEV)
    for s in range(0, X.nnz, 2_000_000):
        c = coords[:, s:s + 2_000_000]
        h = [U[m][c[m]].double() for m in range(X.ndim)]
        model = torch.stack(h).prod(0).sum(1)
        w = vals[s:s + 2_000_000].double() / model.clamp_min(eps)
        want.index_add_(0, c[mode], w[:, None] * torch.stack([h[m] for m in range(X.ndim) if m != mode]).prod(0))
        del h, model, w
    err = (got.double() - want).abs().amax(1) / want.abs().amax(1).clamp_min(1e-30)
    worst = float(err.max())
    del want, err
    pick = np.sort(np.random.default_rng(seed).choice(rows, sample_rows, replace=False))
    return {"vs": f"fp64 device evaluation of every row (max |x - x64| / max |x64| <= 1e-4) + {sample_rows} sampled "
                  "rows bit-compared with the CPU restatement of the order (tests/_cp_apr_order.py)",
            "values_close": worst <= 1e-4, "worst_row_rel_err": worst,
            "sampled_rows_bit_exact": CA.sampled_rows_exact(got, coords, vals, U, mode, pick, 512, eps)}


def _phi_compare(X, U, mode, eps, card):
    """The fused call against (a) the two-launch composition on X's cached stream (Kn.tttp of the stream with the
    values 1, a device clamp and divide, Kn.mttkrp_mode) and (b) the public composed route (tttp on X's pattern, a
    divide of the data, mttkrp_mode on a new COO, which sorts its own mode stream), timed alternately."""
    from sparse_b200 import _fused as F
    from sparse_b200 import _kernels as Kn

    R = U[0].shape[1]
    coords_s, vals_s = F._mode_stream(X, mode)
    ones = torch.ones_like(vals_s)
    rows = X.shape[mode]
    coords, vals = X._dev()
    P = sp.COO(coords, torch.ones_like(vals), shape=X.shape, has_duplicates=False, sorted=True)

    def fused():
        return sp.cp_apr_phi_mode(X, U, mode, eps)

    def two_launch():
        m = Kn.tttp(coords_s, ones, U, R)
        return Kn.mttkrp_mode(coords_s, vals_s / torch.where(m < eps, torch.full_like(m, eps), m), U, mode, rows, R)

    def composed():
        M = sp.tttp(P, U)
        W = sp.COO(coords, vals / M._dev()[1].clamp_min(eps), shape=X.shape, has_duplicates=False, sorted=True)
        return sp.mttkrp_mode(W, U, mode)

    out = {"card": card}
    a, b, c = fused(), two_launch(), composed()
    out["two_launch_bit_equal_to_fused"] = bool(torch.equal(a.view(torch.int32), b.view(torch.int32)))
    out["composed_max_rel_diff_vs_fused"] = float(((c.double() - a.double()).abs().amax(1)
                                                    / a.double().abs().amax(1).clamp_min(1e-30)).max())
    del a, b, c
    for name, f in (("fused", fused), ("two_launch", two_launch), ("composed", composed)):
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats(DEV)
        base = torch.cuda.memory_allocated(DEV)
        f()
        torch.cuda.synchronize()
        out[f"peak_extra_bytes_torch_{name}"] = int(torch.cuda.max_memory_allocated(DEV) - base)
    ms = _alternate({"fused": fused, "two_launch": two_launch, "composed": composed})
    out.update({f"ms_median_{k}": v for k, v in ms.items()})
    out["two_launch_over_fused"] = round(ms["two_launch"] / ms["fused"], 3)
    out["composed_over_fused"] = round(ms["composed"] / ms["fused"], 3)
    return out


def _cp_apr(rec, parity):
    """CP-APR's ratio MTTKRP on the CP-ALS workload of mttkrp_mode ((1e6, 1e6, 100), nnz 1e8, f32, values in [0, 1)),
    nonnegative factors, R = 16 and 32, modes 0 and 2, the mode stream cached; each next to (a) the two-launch
    composition on the same cached stream and (b) the public composed route; and the same comparison on K9's config
    (1e4, 1e4, 1e3, nnz 1e7, R = 32)."""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    out = {}
    card = _card()
    eps = 1e-10
    shape = (1_000_000, 1_000_000, 100)
    X = rand_coo(shape, 100_000_000, 91, torch.float32)
    for R in (16, 32):
        g = torch.Generator(device=DEV).manual_seed(95 + R)
        U = [torch.rand((s, R), generator=g, device=DEV, dtype=torch.float32) for s in shape]
        for mode in (0, 2):
            name = f"cp_apr_phi_mode order-3 (1e6,1e6,100) nnz 1e8 R={R} mode {mode} f32"
            models = _phi_models(X, mode, R)
            r = rec(name, lambda: sp.cp_apr_phi_mode(X, U, mode, eps), X.nnz, "Gnnz_s", models["bytes"]["total"])
            r.update(models)
            r.update(_phi_compare(X, U, mode, eps, card))
            if parity:
                got = sp.cp_apr_phi_mode(X, U, mode, eps)
                r["parity"] = _phi_parity(X, U, mode, eps, got, 8 if mode == 0 else 2, 96)
                del got
            out[name] = r
            print(name, r, flush=True)
        del U
    del X
    torch.cuda.empty_cache()

    X = rand_coo((10_000, 10_000, 1_000), 10_000_000, 31, torch.float32)
    g = torch.Generator(device=DEV).manual_seed(97)
    U = [torch.rand((s, 32), generator=g, device=DEV, dtype=torch.float32) for s in X.shape]
    name = "cp_apr_phi_mode K9 config (1e4,1e4,1e3) nnz 1e7 R=32 mode 0 f32"
    r = rec(name, lambda: sp.cp_apr_phi_mode(X, U, 0, eps), X.nnz, "Gnnz_s", _phi_models(X, 0, 32)["bytes"]["total"])
    r.update(_phi_models(X, 0, 32))
    r.update(_phi_compare(X, U, 0, eps, card))
    if parity:
        r["parity"] = _phi_parity(X, U, 0, eps, sp.cp_apr_phi_mode(X, U, 0, eps), 8, 98)
    out[name] = r
    print(name, r, flush=True)
    del X, U
    torch.cuda.empty_cache()
    return out


def _sptc_fp64(X, Y, ax, ay):
    """(keys, values) of the contraction in float64 on the device: every X entry joined with the Y entries of its
    contracted key (searchsorted + repeat_interleave), the products summed per result key with index_add_."""
    free_x = [a for a in range(X.ndim) if a not in ax]
    free_y = [a for a in range(Y.ndim) if a not in ay]

    def key(c, shape, axes):
        k = torch.zeros(c.shape[1], dtype=torch.int64, device=DEV)
        for a in axes:
            k = k * shape[a] + c[a]
        return k

    xc, xv = X._dev()
    yc, yv = Y._dev()
    g_ext = int(np.prod([Y.shape[a] for a in free_y], dtype=object))
    yC, order = torch.sort(key(yc, Y.shape, ay), stable=True)
    yG, yv = key(yc, Y.shape, free_y)[order], yv[order].double()
    xC, xF = key(xc, X.shape, ax), key(xc, X.shape, free_x)
    lo, hi = torch.searchsorted(yC, xC), torch.searchsorted(yC, xC, right=True)
    cnt = hi - lo
    src = torch.repeat_interleave(torch.arange(xC.numel(), device=DEV), cnt)
    off = torch.arange(src.numel(), device=DEV) - torch.repeat_interleave(torch.cumsum(cnt, 0) - cnt, cnt)
    tgt = lo[src] + off
    keys, inv = torch.unique(xF[src] * g_ext + yG[tgt], return_inverse=True)
    vals = torch.zeros(keys.numel(), dtype=torch.float64, device=DEV).index_add_(0, inv, xv.double()[src] * yv[tgt])
    return keys, vals, int(src.numel())


def _sptc_parity(X, Y, ax, ay, got, sample_rows, seed):
    """Every value against the fp64 device restatement, and `sample_rows` result rows (free keys of X) bit-compared with
    the CPU restatement of the contract (tests/_sptc_order.py)."""
    import _sptc_order as SO

    keys, vals, products = _sptc_fp64(X, Y, ax, ay)
    gk, gv = got.sorted_keys(), got._data_dev()
    pos = torch.searchsorted(keys, gk).clamp_(max=max(keys.numel() - 1, 0))
    present = bool((keys[pos] == gk).all())
    w = vals[pos]
    close = present and bool(torch.allclose(gv.double(), w, rtol=2e-5, atol=2e-5 * float(w.abs().max())))
    free_y = [a for a in range(Y.ndim) if a not in ay]
    g_ext = int(np.prod([Y.shape[a] for a in free_y], dtype=object))
    rows = torch.unique(torch.div(gk, g_ext, rounding_mode="floor"))
    rng = np.random.default_rng(seed)
    pick = rows[torch.from_numpy(np.sort(rng.choice(rows.numel(), min(sample_rows, rows.numel()), replace=False))).to(DEV)]
    xc, xv = X._dev()
    free_x = [a for a in range(X.ndim) if a not in ax]
    xF = torch.zeros(X.nnz, dtype=torch.int64, device=DEV)
    for a in free_x:
        xF = xF * X.shape[a] + xc[a]
    xsel = torch.isin(xF, pick)
    xC = torch.zeros(X.nnz, dtype=torch.int64, device=DEV)
    for a in ax:
        xC = xC * X.shape[a] + xc[a]
    yc, yv = Y._dev()
    yC = torch.zeros(Y.nnz, dtype=torch.int64, device=DEV)
    for a in ay:
        yC = yC * Y.shape[a] + yc[a]
    ysel = torch.isin(yC, torch.unique(xC[xsel]))
    rk, rv = SO.result(xc[:, xsel].cpu().numpy(), xv[xsel].cpu().numpy(), X.shape, yc[:, ysel].cpu().numpy(),
                       yv[ysel].cpu().numpy(), Y.shape, ax, ay, got.dtype)
    gsel = torch.isin(torch.div(gk, g_ext, rounding_mode="floor"), pick)
    exact = bool(np.array_equal(gk[gsel].cpu().numpy(), rk) and SO.same_bits(gv[gsel].cpu().numpy(), rv))
    return {"vs": "fp64 device restatement (rtol 2e-5 of the largest value) and sampled result rows bit-compared with "
                  "tests/_sptc_order.py", "values_close": close, "sampled_rows": int(pick.numel()),
            "sampled_rows_bit_exact": exact}, products


def _sptc_stages(X, Y, ax, ay):
    """ms of the stages of one cached call, each between device synchronisations: the join, K4, the result keys."""
    from sparse_b200 import _fused as F
    from sparse_b200 import _kernels as Kn

    free_x = [a for a in range(X.ndim) if a not in ax]
    free_y = [a for a in range(Y.ndim) if a not in ay]
    xrows, xptr, xcon, xvals = F._sptc_stream(X, free_x, ax, "x", True)
    yrows, yptr, ycols, yrank, yvals = F._sptc_stream(Y, free_y, ay, "y", True)
    g_ext = int(np.prod([Y.shape[a] for a in free_y], dtype=object))
    nF, nC, nG = int(xrows.shape[0]), int(yrows.shape[0]), int(ycols.shape[0])
    joined = Kn.sptc_join(xcon, yrows, np.int32)
    k4 = lambda: Kn.spgemm(xptr, joined, xvals, yptr, yrank, yvals, nF, nC + 1, nG, sorted_order=True, prune=True,
                           want_indptr=False, want_rows=True)
    _, cols, rows, _, _ = k4()
    t = _alternate({"join": lambda: Kn.sptc_join(xcon, yrows, np.int32), "k4": k4,
                    "keys": lambda: Kn.sptc_keys(rows, cols, xrows, ycols, g_ext)})
    return {"stage_ms_median": t, "nF": nF, "nC": nC, "nG": nG}


def _sptc(rec, parity):
    """Sparse x sparse tensor contraction.  Where tensordot fits, sptc and tensordot(return_type=COO) alternating with
    both calls' peak extra device memory and a bit comparison; a hypersparse pair that tensordot cannot take, with the
    first call (stream build), the cached call, its stages and the byte model of the two new kernels."""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    out = {}
    card = _card()

    X = rand_coo((10_000, 1_000, 1_000), 10_000_000, 101, torch.float32)
    Y = rand_coo((1_000, 1_000, 64), 1_000_000, 102, torch.float32)
    ax, ay = [1, 2], [0, 1]
    fns = {"sptc": lambda: sp.sptc(X, Y, (ax, ay)), "tensordot": lambda: sp.tensordot(X, Y, (ax, ay), return_type=sp.COO)}
    peak = {}
    for k, fn in fns.items():
        fn()
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats(DEV)
        base = torch.cuda.memory_allocated(DEV)
        fn()
        torch.cuda.synchronize()
        peak[k] = int(torch.cuda.max_memory_allocated(DEV) - base)
    t = _alternate(fns)
    got, want = fns["sptc"](), fns["tensordot"]()
    name = "sptc (1e4,1e3,1e3) nnz 1e7 . (1e3,1e3,64) nnz 1e6 over two modes f32 vs tensordot(return_type=COO)"
    r = {"ms_median": t["sptc"], "tensordot_ms_median": t["tensordot"],
         "speedup_vs_tensordot": round(t["tensordot"] / t["sptc"], 2), "peak_extra_bytes_streams_cached": peak["sptc"],
         "tensordot_peak_extra_bytes": peak["tensordot"], "out_nnz": got.nnz, "card": card,
         **_sptc_stages(X, Y, ax, ay),
         "whole_result_bit_exact_vs_tensordot": bool(
             got.nnz == want.nnz and torch.equal(got.sorted_keys(), want.sorted_keys())
             and torch.equal(got._data_dev().view(torch.int32), want._data_dev().view(torch.int32)))}
    print(name, r, flush=True)
    out[name] = r
    del X, Y, got, want
    torch.cuda.empty_cache()

    # hypersparse: the matricised X has 1e12 rows and the contracted extent is 1e6; sizes chosen so that the result
    # (about two products per X entry) stays near 4e7 entries
    X = rand_coo((1_000_000,) * 3, 20_000_000, 103, torch.float32)
    Y = rand_coo((1_000_000, 100_000), 2_000_000, 104, torch.float32)
    ax, ay = [2], [0]
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    got = sp.sptc(X, Y, (ax, ay))
    torch.cuda.synchronize()
    first = (time.perf_counter() - t0) * 1e3
    name = "sptc hypersparse (1e6,1e6,1e6) nnz 2e7 . (1e6,1e5) nnz 2e6 over the last mode f32"
    r = rec(name, lambda: sp.sptc(X, Y, (ax, ay)), X.nnz, "Gnnz_s")
    st = _sptc_stages(X, Y, ax, ay)
    model = {"join_bytes": X.nnz * (8 + 4) + st["nC"] * 8, "keys_bytes": got.nnz * (16 + 8)}
    r.update({"card": card, "first_call_ms_incl_streams": round(first, 3), "out_nnz": got.nnz, **st,
              "model_bytes": model,
              "model_join_GBs": round(model["join_bytes"] / st["stage_ms_median"]["join"] / 1e6, 1),
              "model_keys_GBs": round(model["keys_bytes"] / st["stage_ms_median"]["keys"] / 1e6, 1)})
    if parity:
        r["parity"], r["products"] = _sptc_parity(X, Y, ax, ay, got, 2_000, 105)
    print(name, r, flush=True)
    out[name] = r
    del X, Y, got
    torch.cuda.empty_cache()
    return out


def main():
    res = run(sys.argv[1:] or None)
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
