"""sb2_csr_gram (G = X^T X in float64) against float64 truth on every route (need an H100: `pytest -m gpu`).

For rows whose columns strictly increase, csrc/pca.cu sorts the CSR positions by (row chunk, column) and accumulates each
G row in per-warp shared-memory copies (csr_gram_rows_kernel); an unsorted row, or a g whose two warp copies do not fit
in shared memory, takes the one-RED-per-product csr_gram_kernel.  Each case checks every cell to rtol 1e-12 with the
zero pattern of the truth, and the route through the launch count.
"""
import numpy as np
import pytest
import torch
from scipy import sparse

import scanpy_b200 as sb
from scanpy_b200 import _ops

pytestmark = pytest.mark.gpu

# launches per sb2_csr_gram call: count + scan (3) + scatter + rows + mirror; count + plain kernel + mirror when a row is
# unsorted; plain kernel + mirror past the shared-memory limit
ROWS, UNSORTED, PLAIN = 7, 3, 2


def _csr(n, g, density, seed, *, empty_every=0, full_row=None, every_row_col=None, reverse_row=None):
    rs = np.random.RandomState(seed)
    mask = rs.random_sample((n, g)) < density
    if empty_every:
        mask[::empty_every] = False
    if full_row is not None:
        mask[full_row] = True
    if every_row_col is not None:
        mask[:, every_row_col] = True
    x = sparse.csr_matrix(np.where(mask, rs.uniform(0.1, 3.0, (n, g)), 0.0).astype(np.float32))
    x.indptr = x.indptr.astype(np.int64)
    if reverse_row is not None:
        a, b = x.indptr[reverse_row], x.indptr[reverse_row + 1]
        x.indices[a:b] = x.indices[a:b][::-1].copy()
        x.data[a:b] = x.data[a:b][::-1].copy()
    return x


def _gram(x):
    n, g = x.shape
    ctx = sb._abi.default_context()
    dp, di, dd = _ops.csr_to_device(x)
    gram = torch.empty((g, g), dtype=torch.float64, device="cuda")
    torch.cuda.synchronize()
    l0 = ctx.lib.sb2_ctx_launch_count(ctx.handle)
    sb._abi.check(ctx.lib.sb2_csr_gram(ctx.handle, n, g, _ops.ptr(dp), _ops.ptr(di), _ops.ptr(dd), _ops.ptr(gram)))
    torch.cuda.synchronize()
    return gram, ctx.lib.sb2_ctx_launch_count(ctx.handle) - l0


def _truth(x):
    xd = x.astype(np.float64)
    ref = (xd.T @ xd).tocoo()
    out = torch.zeros(x.shape[1], x.shape[1], dtype=torch.float64, device="cuda")
    out[torch.from_numpy(ref.row.astype(np.int64)).cuda(), torch.from_numpy(ref.col.astype(np.int64)).cuda()] = \
        torch.from_numpy(ref.data).cuda()
    return out


CASES = {
    "g1": (lambda: _csr(3000, 1, 0.5, 1), ROWS),
    "g63": (lambda: _csr(5000, 63, 0.1, 2), ROWS),
    "g64": (lambda: _csr(5000, 64, 0.1, 3), ROWS),
    # empty rows, one row holding every gene (nnz_r = g) and a gene stored in every row
    "g2000": (lambda: _csr(20000, 2000, 0.05, 4, empty_every=7, full_row=100, every_row_col=17), ROWS),
    "g8192": (lambda: _csr(3000, 8192, 0.03, 5), ROWS),
    "all_empty": (lambda: _csr(3000, 300, 0.0, 6), ROWS),
    # ~7 KB per row: several row chunks, the last one partial, and gene 0 in every row of each
    "chunks": (lambda: _csr(9000, 1000, 0.9, 7, every_row_col=0), ROWS),
    "unsorted": (lambda: _csr(4000, 500, 0.06, 8, reverse_row=2000), UNSORTED),
    # two fp64 copies of a G row take 256 KB, more than a CTA's shared memory
    "g16000": (lambda: _csr(256, 16000, 0.02, 9), PLAIN),
}


@pytest.mark.parametrize("name", list(CASES))
def test_gram_against_f64(name):
    make, route = CASES[name]
    x = make()
    gram, launches = _gram(x)
    ref = _truth(x)
    nz = ref != 0
    assert bool(((gram != 0) == nz).all()), "zero pattern differs from the truth"
    rel = float(((gram - ref).abs()[nz] / ref[nz].abs()).max()) if bool(nz.any()) else 0.0
    print(f"\n[gram {name}] {x.shape[0]} x {x.shape[1]}, nnz {x.nnz}: max rel err {rel:.1e} (bar 1e-12), "
          f"{launches} launches")
    assert rel <= 1e-12
    assert launches == route, (launches, route)


def test_gram_repeatable():
    # the fp64 sums are taken in a different order from call to call (shared-memory ranks, REDs), never by more than
    # the last bits
    x = _csr(20000, 2000, 0.05, 10)
    g1, _ = _gram(x)
    g2, _ = _gram(x)
    diff = float((g1 - g2).abs().max() / g1.abs().max())
    print(f"\n[gram repeat] max |G1 - G2| / max |G1| = {diff:.1e} (bar 1e-15)")
    assert diff <= 1e-15
