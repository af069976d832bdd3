"""pp.bsr_bsc_matmul and pp.sparse (csrc/bsr.cu, csrc/bsr_math.cuh) against reference goldens
(oracle/make_golden_sparse.py), the numpy oracle (oracle/sparse_oracle.py) and a host build of the accumulation
(tests/sparse_host.cpp).  DESIGN.md §3.8."""
import ctypes
import json
import os
import subprocess
import tempfile
import warnings

import numpy as np
import pytest
import torch

import pypose_b200 as pp
from pypose_b200.sparse.ops import _sparse_csr_mm, _BsrBscValues
from oracle import sparse_oracle as O

warnings.filterwarnings("ignore", message=".*Sparse.*")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = np.load(os.path.join(ROOT, "tests", "golden", "sparse.npz"))
NAMES = json.loads(str(GOLD["cases"]))
DEV = torch.device("cuda:0")
_HOST = {}


def g(name, k):
    return GOLD[f"{name}/{k}"]


def golden_operands(name, dev="cpu", idx_dtype=torch.int64):
    a_size, b_size = tuple(int(x) for x in g(name, "a_size")), tuple(int(x) for x in g(name, "b_size"))
    t = lambda k, dt=None: torch.from_numpy(np.ascontiguousarray(g(name, k))).to(dev, dt)   # noqa: E731
    A = torch.sparse_bsr_tensor(t("a_crow", idx_dtype), t("a_col", idx_dtype), t("a_val"), size=a_size)
    B = torch.sparse_bsc_tensor(t("b_ccol", idx_dtype), t("b_row", idx_dtype), t("b_val"), size=b_size)
    return A, B


def grids(name):
    a_val, b_val = g(name, "a_val"), g(name, "b_val")
    a_size, b_size = g(name, "a_size"), g(name, "b_size")
    return a_size[0] // a_val.shape[1], b_size[1] // b_val.shape[2]


def rel_close(a, b, tol):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.abs(a - b).max(initial=0.0) <= tol * (1 + np.abs(b).max(initial=0.0))


def _host():
    if "lib" not in _HOST:
        d = tempfile.mkdtemp(prefix="sparse_host_")
        so = os.path.join(d, "libsparsehost.so")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC",
                               "-I", os.path.join(ROOT, "pypose_b200", "csrc"), os.path.join(ROOT, "tests", "sparse_host.cpp"),
                               "-o", so])
        _HOST["lib"] = ctypes.CDLL(so)
    return _HOST["lib"]


def host_numeric(L, lstr, R, rstr, tri, ptr, dx, dy, dz):
    """out (nout, dx, dy) of the host build; L / R are flat arrays read through the element strides lstr / rstr"""
    dt = L.dtype
    tri = np.ascontiguousarray(tri, np.uint64)
    ptr = np.ascontiguousarray(ptr, np.int64)
    out = np.empty((len(ptr) - 1, dx, dy), dt)
    f = getattr(_host(), "sparse_host_numeric_" + ("f64" if dt == np.float64 else "f32"))
    vp = lambda a: ctypes.c_void_p(a.ctypes.data)   # noqa: E731
    ll = ctypes.c_longlong
    f(vp(L), *[ll(s) for s in lstr], vp(R), *[ll(s) for s in rstr], vp(tri), vp(ptr), ll(len(ptr) - 1),
      ctypes.c_int(dx), ctypes.c_int(dy), ctypes.c_int(dz), vp(out))
    return out


def host_product(a_crow, a_col, a_val, b_ccol, b_row, b_val, sp):
    """C's values from the host build in the device's order: triples (a << 32) | b in (i, j, k) order"""
    key, a, b = O.triples(a_crow, a_col, b_ccol, b_row, sp)
    _, start = np.unique(key, return_index=True)
    ptr = np.append(start, len(key))
    A, B = np.ascontiguousarray(a_val), np.ascontiguousarray(b_val)
    es = A.itemsize
    tri = (a.astype(np.uint64) << np.uint64(32)) | b.astype(np.uint64)
    return host_numeric(A, [s // es for s in A.strides], B, [s // es for s in B.strides], tri, ptr, A.shape[1],
                        B.shape[2], A.shape[2])


# ------------------------------------------------------------------------------------------------------------- CPU
@pytest.mark.parametrize("name", NAMES)
def test_oracle_reproduces_reference_goldens(name):
    sm, sp = grids(name)
    crow, col, val = O.product(g(name, "a_crow"), g(name, "a_col"), g(name, "a_val"), g(name, "b_ccol"), g(name, "b_row"),
                               g(name, "b_val"), sm, sp)
    np.testing.assert_array_equal(crow, g(name, "crow"))
    np.testing.assert_array_equal(col, g(name, "col"))
    assert rel_close(val, g(name, "val"), 1e-12 if g(name, "val").dtype == np.float64 else 1e-5)


@pytest.mark.parametrize("name", [n for n in NAMES if "f64" in n])
def test_host_build_reproduces_reference_goldens(name):
    sm, sp = grids(name)
    val = host_product(g(name, "a_crow"), g(name, "a_col"), g(name, "a_val"), g(name, "b_ccol"), g(name, "b_row"),
                       g(name, "b_val"), sp)
    assert val.shape == g(name, "val").shape and rel_close(val, g(name, "val"), 1e-12)


def test_host_build_reads_transposed_strides():
    rng = np.random.default_rng(3)
    crow, col, val = O.random_bsr(30, 20, 3, 5, 0.2, rng)
    ccol, row, bval = O.transpose_pattern(crow, col, val)          # a (5, 3) view over A's blocks
    assert not bval.flags.c_contiguous
    key, a, b = O.triples(crow, col, ccol, row, 30)
    _, start = np.unique(key, return_index=True)
    tri = (a.astype(np.uint64) << np.uint64(32)) | b.astype(np.uint64)
    out = host_numeric(val, [15, 5, 1], val, [15, 1, 5], tri, np.append(start, len(key)), 3, 3, 5)
    _, _, want = O.product(crow, col, val, ccol, row, bval, 30, 30)
    assert rel_close(out, want, 1e-13)


def _bsr(sm, sn, dm, dn, seed=0, dtype=torch.float64, dev="cpu"):
    crow, col, val = O.random_bsr(sm, sn, dm, dn, 0.5, np.random.default_rng(seed))
    return torch.sparse_bsr_tensor(torch.from_numpy(crow), torch.from_numpy(col), torch.from_numpy(val).to(dtype),
                                   size=(sm * dm, sn * dn)).to(dev)


def test_argument_errors():
    A = _bsr(4, 3, 2, 5)
    B = _bsr(3, 4, 5, 2).to_dense().to_sparse_bsc((5, 2))
    with pytest.raises(NotImplementedError):
        pp.bsr_bsc_matmul(B, A)
    with pytest.raises(ValueError):                                  # layouts
        pp.bsr_bsc_matmul(A, B.to_dense())
    with pytest.raises(ValueError):
        pp.bsr_bsc_matmul(A.to_dense().to_sparse_csr(), B)
    with pytest.raises(ValueError):
        pp.bsr_bsc_matmul(A, A.mT.to_dense().to_sparse_bsr((5, 2)))
    with pytest.raises(ValueError):                                  # dtype mix
        pp.bsr_bsc_matmul(A, B.to(torch.float32))
    with pytest.raises(ValueError):                                  # unsupported dtype
        pp.bsr_bsc_matmul(A.to(torch.float16), B.to(torch.float16))
    with pytest.raises(ValueError):                                  # inner block size mismatch
        pp.bsr_bsc_matmul(A, B.to_dense().to_sparse_bsc((3, 2)))
    with pytest.raises(ValueError):                                  # inner size mismatch
        pp.bsr_bsc_matmul(A, _bsr(4, 4, 5, 2).to_dense().to_sparse_bsc((5, 2)))
    with pytest.raises(ValueError):                                  # batch dimension
        pp.bsr_bsc_matmul(torch.stack([A.to_dense()] * 2).to_sparse_bsr((2, 5)), B)
    one = torch.ones(1, 2, 5, dtype=torch.float64)
    bad = torch.sparse_bsr_tensor(torch.tensor([0, 1]), torch.tensor([0]), one, size=(3, 5), check_invariants=False)
    with pytest.raises(ValueError):                                  # shape not divisible by the blocks
        pp.bsr_bsc_matmul(bad, torch.sparse_bsc_tensor(torch.tensor([0, 1]), torch.tensor([0]), one.mT, size=(5, 2)))
    with pytest.raises(NotImplementedError, match="CPU"):            # no CPU path
        pp.bsr_bsc_matmul(A, B)
    with pytest.raises(NotImplementedError):
        _sparse_csr_mm(B, A)


def test_public_names():
    assert pp.bsr_bsc_matmul is pp.sparse.bsr_bsc_matmul
    from pypose_b200.sparse import ops
    assert ops._sparse_csr_mm is _sparse_csr_mm


@pytest.mark.parametrize("l1", ["csr", "csc", "strided"])
@pytest.mark.parametrize("l2", ["csr", "csc", "strided"])
def test_sparse_csr_mm_routes_non_block_layouts_to_torch(l1, l2):
    gen = torch.Generator().manual_seed(5)
    d, e = torch.randn(7, 9, generator=gen, dtype=torch.float64), torch.randn(9, 6, generator=gen, dtype=torch.float64)
    d[d < 0.3], e[e < 0.3] = 0, 0
    conv = {"csr": lambda t: t.to_sparse_csr(), "csc": lambda t: t.to_sparse_csc(), "strided": lambda t: t}
    out = _sparse_csr_mm(conv[l1](d), conv[l2](e))
    want_layout = torch.strided if l2 == "strided" or l1 == "strided" else torch.sparse_csr
    assert out.layout == want_layout
    torch.testing.assert_close(out.to_dense() if out.layout != torch.strided else out, d @ e, rtol=1e-14, atol=1e-14)


def test_sparse_csr_mm_routes_bsr_times_strided_to_torch():
    A = _bsr(4, 3, 3, 3)                                             # torch's CPU BSR product takes square blocks
    e = torch.randn(9, 4, dtype=torch.float64)
    torch.testing.assert_close(_sparse_csr_mm(A, e), A.to_dense() @ e, rtol=1e-14, atol=1e-14)


# ------------------------------------------------------------------------------------------------------------- GPU
def to_np(C):
    return C.crow_indices().cpu().numpy(), C.col_indices().cpu().numpy(), C.values().detach().cpu().numpy()


@pytest.mark.gpu
@pytest.mark.parametrize("idx_dtype", [torch.int64, torch.int32])
@pytest.mark.parametrize("name", NAMES)
def test_goldens(name, idx_dtype):
    A, B = golden_operands(name, DEV, idx_dtype)
    for C in (pp.bsr_bsc_matmul(A, B), _sparse_csr_mm(A, B)):
        assert C.layout == torch.sparse_bsr and C.shape == (A.shape[0], B.shape[1]) and C.device == A.device
        assert C.crow_indices().dtype == torch.int64 and C.col_indices().dtype == torch.int64
        crow, col, val = to_np(C)
        np.testing.assert_array_equal(crow, g(name, "crow"))
        np.testing.assert_array_equal(col, g(name, "col"))
        assert val.dtype == g(name, "val").dtype and val.shape == g(name, "val").shape
        assert rel_close(val, g(name, "val"), 1e-12 if val.dtype == np.float64 else 1e-5)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("shape", [(40, 30, 50, 3, 6, 4, 0.3), (200, 150, 120, 1, 1, 1, 0.05), (60, 60, 60, 9, 9, 9, 0.1),
                                   (300, 200, 250, 2, 7, 3, 0.02)])
def test_random_against_oracle_and_host_build(shape, dtype):
    sm, sn, sp, dm, dn, dp, dens = shape
    rng = np.random.default_rng(sm + sn + dm)
    a = O.random_bsr(sm, sn, dm, dn, dens, rng, dtype=dtype)
    bt = O.random_bsr(sp, sn, dp, dn, dens, rng, dtype=dtype)        # B^T in BSR = B in BSC with transposed blocks
    b = O.transpose_pattern(*bt)
    A = torch.sparse_bsr_tensor(*[torch.from_numpy(np.ascontiguousarray(x)) for x in a], size=(sm * dm, sn * dn)).to(DEV)
    B = torch.sparse_bsc_tensor(*[torch.from_numpy(np.ascontiguousarray(x)) for x in b], size=(sn * dn, sp * dp)).to(DEV)
    C = pp.bsr_bsc_matmul(A, B)
    crow, col, val = to_np(C)
    wc, wl, wv = O.product(*a, *b, sm, sp)
    np.testing.assert_array_equal(crow, wc)
    np.testing.assert_array_equal(col, wl)
    assert rel_close(val, wv, 1e-12 if dtype == np.float64 else 1e-5)
    assert np.array_equal(val, host_product(*a, *b, sp))             # bit for bit
    val2 = to_np(pp.bsr_bsc_matmul(A, B))[2]
    assert np.array_equal(val, val2)                                  # repeated calls


@pytest.mark.gpu
def test_large_pattern_1e5_block_rows():
    """A @ A.mT on a 1e5 × 1e5 grid of 2 × 2 blocks, 10 blocks per row: about 1e7 block products."""
    n, per = 100000, 10
    rng = np.random.default_rng(11)
    col = np.sort(np.stack([rng.choice(n, per, replace=False) for _ in range(64)]), 1)   # reused row patterns
    col = col[rng.integers(0, 64, n)] + rng.integers(0, n, (n, 1))
    col = np.sort(col % n, 1)
    keep = np.concatenate([np.ones((n, 1), bool), np.diff(col, axis=1) > 0], 1)
    cnt = keep.sum(1)
    crow = np.concatenate([[0], np.cumsum(cnt)]).astype(np.int64)
    col = col[keep].astype(np.int64)
    val = rng.standard_normal((len(col), 2, 2))
    A = torch.sparse_bsr_tensor(torch.from_numpy(crow), torch.from_numpy(col), torch.from_numpy(val), size=(2 * n, 2 * n))
    A = A.to(DEV)
    C = pp.bsr_bsc_matmul(A, A.mT)
    ccol, row, bval = O.transpose_pattern(crow, col, val)
    key, _, _ = O.triples(crow, col, ccol, row, n)
    assert len(key) > 8e6
    wc, wl = O.pattern(crow, col, ccol, row, n, n)
    crow_g, col_g = C.crow_indices().cpu().numpy(), C.col_indices().cpu().numpy()
    np.testing.assert_array_equal(crow_g, wc)
    np.testing.assert_array_equal(col_g, wl)
    rows = np.sort(rng.choice(n, 200, replace=False))
    _, _, wv = O.product(crow, col, val, ccol, row, bval, n, n, rows=rows)
    got = C.values().cpu().numpy()[np.concatenate([np.arange(wc[r], wc[r + 1]) for r in rows])]
    assert rel_close(got, wv, 1e-12)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
def test_a_at_with_int32_indices_and_strided_values(dtype):
    rng = np.random.default_rng(4)
    crow, col, val = O.random_bsr(50, 40, 3, 4, 0.15, rng)
    big = torch.from_numpy(rng.standard_normal((len(col), 6, 9))).to(DEV, dtype)
    v = big[:, ::2, 1::2][:, :, :4]                                   # (nnz, 3, 4), strided in every axis
    v.copy_(torch.from_numpy(val))
    assert not v.is_contiguous()
    A = torch.sparse_bsr_tensor(torch.from_numpy(crow).int().to(DEV), torch.from_numpy(col).int().to(DEV), v,
                                size=(150, 160))
    assert not A.values().is_contiguous() and A.crow_indices().dtype == torch.int32
    C = pp.bsr_bsc_matmul(A, A.mT)
    assert not A.mT.values().is_contiguous()
    wc, wl, wv = O.product(crow, col, val, *O.transpose_pattern(crow, col, val), 50, 50)
    crow_g, col_g, got = to_np(C)
    np.testing.assert_array_equal(crow_g, wc)
    np.testing.assert_array_equal(col_g, wl)
    assert rel_close(got, wv, 1e-12 if dtype == torch.float64 else 1e-5)
    assert np.array_equal(got, host_product(crow, col, val.astype(got.dtype), *O.transpose_pattern(crow, col,
                                                                                                    val.astype(got.dtype)), 50))
    torch.testing.assert_close(C.to_dense(), A.to_dense() @ A.to_dense().mT)


@pytest.mark.gpu
def test_empty_results():
    d = torch.float64
    z = lambda n: torch.zeros(n + 1, dtype=torch.int64)   # noqa: E731
    A0 = torch.sparse_bsr_tensor(z(5), torch.zeros(0, dtype=torch.int64), torch.zeros(0, 2, 3, dtype=d), size=(10, 12)).to(DEV)
    B = _bsr(4, 4, 2, 3).mT.to(DEV)                                  # (12, 8) BSC with (3, 2) blocks
    for A_, B_ in ((A0, B), (_bsr(5, 4, 2, 3).to(DEV), torch.sparse_bsc_tensor(z(4), torch.zeros(0, dtype=torch.int64),
                                                                               torch.zeros(0, 3, 2, dtype=d),
                                                                               size=(12, 8)).to(DEV))):
        C = pp.bsr_bsc_matmul(A_, B_)
        assert C.layout == torch.sparse_bsr and C.shape == (10, 8) and C.values().shape == (0, 2, 2)
        assert C.crow_indices().tolist() == [0] * 6 and C.to_dense().abs().sum() == 0
    A = torch.zeros(10, 12, dtype=d)
    A[:, :3] = 1.0                                                   # block column 0 only
    Bd = torch.zeros(12, 8, dtype=d)
    Bd[3:, :] = 1.0                                                  # block rows 1..3 only
    C = pp.bsr_bsc_matmul(A.to_sparse_bsr((2, 3)).to(DEV), Bd.to_sparse_bsc((3, 2)).to(DEV))
    assert C.values().shape == (0, 2, 2) and C.crow_indices().tolist() == [0] * 6


def values_product(va, vb, a_crow, a_col, b_ccol, b_row, sm, sn, sp):
    """C's values through the module's autograd Function over the values (vb None: B = A.mT)"""
    return _BsrBscValues.apply(va, vb, a_crow, a_col, b_ccol, b_row, sm, sn, sp)[0]


def _grad_operands(dtype=torch.float64, seed=1):
    rng = np.random.default_rng(seed)
    a = [torch.from_numpy(x).to(DEV) for x in O.random_bsr(7, 6, 2, 3, 0.4, rng)]
    b = [torch.from_numpy(x).to(DEV) for x in O.random_bsr(5, 6, 4, 3, 0.4, rng)]
    va = a[2].to(dtype).requires_grad_()
    vb = b[2].to(dtype).mT.contiguous().requires_grad_()              # (nnz, 3, 4) blocks of B in BSC
    return (lambda x, y: values_product(x, y, a[0], a[1], b[0], b[1], 7, 6, 5)), va, vb, a, b


@pytest.mark.gpu
def test_gradcheck_fp64():
    f, va, vb, _, _ = _grad_operands()
    assert torch.autograd.gradcheck(f, (va, vb))
    assert torch.autograd.gradcheck(lambda x: f(x, vb.detach()), (va,))
    assert torch.autograd.gradcheck(lambda y: f(va.detach(), y), (vb,))
    crow, col, val = (torch.from_numpy(x).to(DEV) for x in O.random_bsr(6, 5, 3, 2, 0.4, np.random.default_rng(8)))
    a_at = lambda v: values_product(v, None, crow, col, crow, col, 6, 5, 6)   # noqa: E731  B = A.mT
    assert torch.autograd.gradcheck(a_at, (val.clone().requires_grad_(),))


@pytest.mark.gpu
def test_gradients_flow_through_the_sparse_constructors():
    """End to end through torch.sparse_bsr_tensor(..., values) / .values(), at a size where torch's own sparse autograd
    (it forms dense (m, p) intermediates) is cheap: the same gradients as the values-level Function."""
    f, va, vb, a, b = _grad_operands(seed=3)
    A = torch.sparse_bsr_tensor(a[0], a[1], va, size=(14, 18))
    B = torch.sparse_bsc_tensor(b[0], b[1], vb, size=(18, 20))
    C = pp.bsr_bsc_matmul(A, B)
    w = torch.randn_like(C.values())
    ga, gb = torch.autograd.grad((C.values() * w).sum(), (va, vb))
    wa, wb = torch.autograd.grad((f(va, vb) * w).sum(), (va, vb))
    torch.testing.assert_close(ga, wa, rtol=1e-13, atol=1e-13)
    torch.testing.assert_close(gb, wb, rtol=1e-13, atol=1e-13)


@pytest.mark.gpu
def test_gradients_of_a_at_and_bit_identical():
    rng = np.random.default_rng(9)
    crow, col, val = O.random_bsr(400, 300, 6, 6, 0.02, rng)
    crow_t, col_t = torch.from_numpy(crow).to(DEV), torch.from_numpy(col).to(DEV)
    v = torch.from_numpy(val).to(DEV).requires_grad_()
    C = values_product(v, None, crow_t, col_t, crow_t, col_t, 400, 300, 400)
    W = torch.randn_like(C)

    def run():
        c = values_product(v, None, crow_t, col_t, crow_t, col_t, 400, 300, 400)
        (gv,) = torch.autograd.grad((c * W).sum(), v)
        return c.detach(), gv
    c1, g1 = run()
    c2, g2 = run()
    assert torch.equal(c1, c2) and torch.equal(g1, g2)
    # d/dA <W, A A^T> = (W + W^T) A on the stored blocks of A
    A = torch.sparse_bsr_tensor(crow_t, col_t, v.detach(), size=(2400, 1800))
    Cs = pp.bsr_bsc_matmul(A, A.mT)
    Wd = torch.sparse_bsr_tensor(Cs.crow_indices(), Cs.col_indices(), W, size=(2400, 2400)).to_dense()
    Gd = (Wd + Wd.T) @ A.to_dense()
    stored = torch.sparse_bsr_tensor(crow_t, col_t, torch.ones_like(v), size=(2400, 1800)).to_dense() != 0
    got = torch.sparse_bsr_tensor(crow_t, col_t, g1, size=(2400, 1800)).to_dense()
    assert torch.allclose(got, Gd * stored, rtol=1e-11, atol=1e-11)


@pytest.mark.gpu
def test_gradients_fp32_match_fp64():
    f64, va, vb, _, _ = _grad_operands(torch.float64, seed=2)
    f32, va32, vb32, _, _ = _grad_operands(torch.float32, seed=2)
    w = torch.randn_like(f64(va, vb))
    ga, gb = torch.autograd.grad((f64(va, vb) * w).sum(), (va, vb))
    ga32, gb32 = torch.autograd.grad((f32(va32, vb32) * w.float()).sum(), (va32, vb32))
    assert rel_close(ga32.cpu().numpy(), ga.cpu().numpy(), 1e-5) and rel_close(gb32.cpu().numpy(), gb.cpu().numpy(), 1e-5)


@pytest.mark.gpu
def test_host_read_budget():
    rng = np.random.default_rng(6)
    crow, col, val = O.random_bsr(2000, 1500, 6, 6, 0.004, rng)
    v = torch.from_numpy(val).to(DEV).requires_grad_()
    crow_t, col_t = torch.from_numpy(crow).to(DEV), torch.from_numpy(col).to(DEV)
    A = torch.sparse_bsr_tensor(crow_t, col_t, v.detach(), size=(12000, 9000))
    pp.bsr_bsc_matmul(A, A.mT)                                       # warm up
    values_product(v, None, crow_t, col_t, crow_t, col_t, 2000, 1500, 2000).sum().backward()
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("warn")
    try:
        with warnings.catch_warnings(record=True) as w_fwd:
            warnings.simplefilter("always")
            A = torch.sparse_bsr_tensor(crow_t, col_t, v.detach(), size=(12000, 9000))
            pp.bsr_bsc_matmul(A, A.mT)
        loss = values_product(v, None, crow_t, col_t, crow_t, col_t, 2000, 1500, 2000).sum()
        with warnings.catch_warnings(record=True) as w_bwd:
            warnings.simplefilter("always")
            loss.backward()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    fwd = [str(x.message) for x in w_fwd if "synchroniz" in str(x.message)]
    bwd = [str(x.message) for x in w_bwd if "synchroniz" in str(x.message)]
    assert len(fwd) == 2, fwd
    assert len(bwd) == 0, bwd


@pytest.mark.gpu
def test_invalid_indices_raise():
    one = torch.ones(2, 2, 2, dtype=torch.float64)
    B = torch.sparse_bsc_tensor(torch.tensor([0, 1, 2]), torch.tensor([0, 1]), one, size=(4, 4)).to(DEV)

    def A(crow, col):
        return torch.sparse_bsr_tensor(torch.tensor(crow), torch.tensor(col), one, size=(4, 4),
                                       check_invariants=False).to(DEV)
    with pytest.raises(ValueError):
        pp.bsr_bsc_matmul(A([0, 2, 2], [0, 2]), B)                   # column out of range
    with pytest.raises(ValueError):
        pp.bsr_bsc_matmul(A([0, 2, 2], [1, 0]), B)                   # unsorted within a row
    with pytest.raises(ValueError):
        pp.bsr_bsc_matmul(A([0, 2, 2], [1, 1]), B)                   # repeated within a row
    with pytest.raises(ValueError):
        pp.bsr_bsc_matmul(A([0, 1, 2], [0, -1]), B)                  # negative
    with pytest.raises(ValueError):
        pp.bsr_bsc_matmul(A([0, 2, 1], [0, 1]), B)                   # decreasing pointers
    bad_b = torch.sparse_bsc_tensor(torch.tensor([0, 2, 2]), torch.tensor([1, 0]), one, size=(4, 4),
                                    check_invariants=False).to(DEV)
    with pytest.raises(ValueError):
        pp.bsr_bsc_matmul(A([0, 1, 2], [0, 1]), bad_b)               # unsorted within a column of B
    C = pp.bsr_bsc_matmul(A([0, 1, 2], [0, 1]), B)                   # still works afterwards
    torch.testing.assert_close(C.to_dense().cpu(), torch.block_diag(torch.full((2, 2), 2.0), torch.full((2, 2), 2.0)).double())


def test_transpose_detection_follows_the_autograd_graph():
    from pypose_b200.sparse.ops import _is_transpose_of
    rng = np.random.default_rng(12)
    crow, col, val = (torch.from_numpy(x) for x in O.random_bsr(5, 4, 2, 3, 0.5, rng))
    v = val.clone().requires_grad_()
    A = torch.sparse_bsr_tensor(crow, col, v, size=(10, 12))
    assert _is_transpose_of(A.mT, A)
    assert not _is_transpose_of(A.detach().mT, A)                   # stop-gradient on B: separate gradients
    assert not _is_transpose_of(A.mT, A.detach())                   # stop-gradient on A
    assert not _is_transpose_of(torch.sparse_bsc_tensor(crow, col, v.detach().mT, size=(12, 10)), A)
    assert not _is_transpose_of(torch.sparse_bsc_tensor(crow, col, v.mT, size=(12, 10)), A)   # another graph node
    D = A.detach()
    assert _is_transpose_of(D.mT, D)                                # no gradients at all
    L = torch.sparse_bsr_tensor(crow, col, val.clone(), size=(10, 12)).requires_grad_()       # a sparse leaf
    assert _is_transpose_of(L.mT, L) and not _is_transpose_of(L.detach().mT, L)


def _small_a(seed):
    crow, col, val = O.random_bsr(12, 9, 3, 2, 0.3, np.random.default_rng(seed))
    crow_t, col_t = torch.from_numpy(crow).to(DEV), torch.from_numpy(col).to(DEV)
    v = torch.from_numpy(val).to(DEV).requires_grad_()
    stored = torch.sparse_bsr_tensor(crow_t, col_t, torch.ones_like(v), size=(36, 18)).to_dense() != 0
    return crow_t, col_t, v, stored


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["both", "detach_b", "detach_a"])
def test_a_at_gradients_through_the_sparse_constructors(mode):
    """pp.bsr_bsc_matmul(A, A.mT), (A, A.detach().mT) and (A.detach(), A.mT) end to end through torch.sparse_bsr_tensor
    and .values(): the gradient of <W, C> with respect to A's values against the dense formula on A's stored blocks."""
    crow_t, col_t, v, stored = _small_a(13)
    A = torch.sparse_bsr_tensor(crow_t, col_t, v, size=(36, 18))
    L, R = {"both": (A, A.mT), "detach_b": (A, A.detach().mT), "detach_a": (A.detach(), A.mT)}[mode]
    C = pp.bsr_bsc_matmul(L, R)
    W = torch.randn_like(C.values())
    (gv,) = torch.autograd.grad((C.values() * W).sum(), v)
    Wd = torch.sparse_bsr_tensor(C.crow_indices(), C.col_indices(), W, size=(36, 36)).to_dense()
    Ad = A.detach().to_dense()
    Gd = {"both": (Wd + Wd.T) @ Ad, "detach_b": Wd @ Ad, "detach_a": Wd.T @ Ad}[mode]
    got = torch.sparse_bsr_tensor(crow_t, col_t, gv, size=(36, 18)).to_dense()
    torch.testing.assert_close(got, Gd * stored, rtol=1e-12, atol=1e-12)
