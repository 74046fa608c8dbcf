"""CPU restatement of the order of operations of cp_apr_phi_mode (include/sparse_b200.h: b2s_cp_apr_phi_mode), built
from the shared restatement of the other sparse-tensor ops in _tensor_order.py: tttp's model values for the values 1,
then the ratios w, then mttkrp_mode of them.

Shared by tests/test_cp_apr_phi_mode.py and the benchmark's parity checks (tools/bench_configs.py).  It imports nothing
from the NumPy stand-in in _mock_cp_apr.py, so a GPU result that matches it means something.  Each operation is a
float32 / float64 NumPy array operation: correctly rounded, and never contracted into an FMA."""
import numpy as np

from _tensor_order import mttkrp_mode, products, row_result, same_bits, values


def ratios(coords, vals, factors, dtype, eps):
    """w_e = v_e / d_e, d_e = eps if m_e < eps else m_e (a NaN m_e stays NaN), with m_e the model of every factor at e:
    tttp's value for the values 1 (1 * m is m)."""
    dtype = np.dtype(dtype)
    m = values(coords, np.ones(np.shape(coords)[1], dtype), factors, dtype)
    e = dtype.type(eps)
    with np.errstate(all="ignore"):
        return np.asarray(vals, dtype=dtype) / np.where(m < e, e, m)


def cp_apr_phi_mode(coords, vals, factors, mode, rows, chunk, dtype, eps):
    """The whole cp_apr_phi_mode result for a tensor given by C-order `coords` (N x nnz) and `vals`."""
    return mttkrp_mode(coords, ratios(coords, vals, factors, dtype, eps), factors, mode, rows, chunk, dtype)


def sampled_rows_exact(got, coords, vals, U, mode, rows, chunk, eps):
    """Whether rows `rows` of the device result `got` equal this restatement bit for bit.  `coords` (N x nnz) and `vals`
    are the tensor's device entries in C order, so a row's entries are in stream order, the first at the stream position
    that counts the entries of the rows before it; the ratios of each row's entries are formed here."""
    import torch

    exact = True
    for i in rows:
        i = int(i)
        sel = torch.nonzero(coords[mode] == i).reshape(-1)
        start = int((coords[mode] < i).sum())
        c = coords[:, sel].cpu().numpy()
        v = vals[sel].cpu().numpy()
        gathered = [U[m][torch.from_numpy(c[m]).to(U[m].device)].cpu().numpy() for m in range(len(U))]
        own = np.tile(np.arange(len(v)), (len(U), 1))  # entry k reads row k of each gathered factor
        w = ratios(own, v, gathered, v.dtype, eps)
        p = products(w, [gathered[m] for m in range(len(U)) if m != mode], v.dtype)
        exact &= same_bits(got[i].cpu().numpy(), row_result(p, start, chunk, v.dtype))
    return bool(exact)
