"""Every kernel path of pp.bsr_bsc_matmul (csrc/bsr.cu, csrc/bsr_math.cuh, sparse/ops.py _BsrBscValues) and of both
gradients against the fp64 oracle (oracle/sparse_oracle.py) and the host build of the accumulation (tests/sparse_host.cpp),
in fp32 and fp64.  DESIGN.md §3.8.

Each product is checked three ways: the pattern (crow, col) and the device's (i, j, k)-ordered triples exactly; the
forward values and dA, dB bit for bit against the host build replaying the oracle's triple orders (the forward order,
and for the gradients the stable regroup by A or B entry); and elementwise against the fp64 oracle within
gamma_n sum |l| |r|, gamma_n = n u / (1 - n u), n = (segment length) dz, the rigorous bound for one fma chain.

Each case asserts the path it is meant to reach: the width of each of bsr.cu's four radix sorts (B's row transpose on
bits_of(sn - 1), the triple keys on bits_of(sm sp - 1), the dA / dB regroups on bits_of(nnzA - 1) / bits_of(nnzB - 1))
with keys on both sides of the top bit, or more output elements than one pass of a grid-stride loop covers (2^20 CTAs of
256 threads).  Not reached here: a second grid-stride pass of the entry, expand, flag and regroup kernels, which needs
more than 2^28 stored blocks or block products (20 GB or more of device memory).
"""
import numpy as np
import pytest
import torch

import pypose_b200 as pp
from pypose_b200 import _C
from pypose_b200.sparse.ops import _BsrBscValues
from oracle import sparse_oracle as O
from tests.test_sparse import host_numeric, values_product

DEV = "cuda"
F32, F64 = torch.float32, torch.float64
PASS = 256 << 20                      # elements one pass of a bsr.cu grid-stride loop covers: kBsMaxGrid x kBsThreads
INT31 = 2 ** 31 - 1


def bits_of(v):
    """bsr.cu bits_of: bits to represent v, at least 1"""
    b = 1
    while b < 64 and v >> b:
        b += 1
    return b


def widths(sm, sn, sp, nnz_a, nnz_b):
    """the radix-sort widths of bsr.cu: B's row transpose, the triple keys, the dA and the dB regroups"""
    return {"brow": bits_of(sn - 1), "key": bits_of(sm * sp - 1), "dA": bits_of(nnz_a - 1), "dB": bits_of(nnz_b - 1)}


def gamma(n, u):
    return n * u / (1 - n * u)


# ---------------------------------------------------------------------------------------------------------------------
# patterns
# ---------------------------------------------------------------------------------------------------------------------
def bsr(rows, cols, sm, dm, dn, rng):
    """(crow, col, values (nnz, dm, dn)) of the BSR matrix with blocks at the (distinct) pairs (rows, cols)"""
    rows, cols = np.asarray(rows, np.int64), np.asarray(cols, np.int64)
    o = np.lexsort((cols, rows))
    return np.searchsorted(rows[o], np.arange(sm + 1)), cols[o], rng.standard_normal((len(o), dm, dn))


def bsc(rows, cols, sp, dn, dp, rng):
    """(ccol, row, values (nnz, dn, dp)) of the BSC matrix with blocks at the (distinct) pairs (rows, cols)"""
    rows, cols = np.asarray(rows, np.int64), np.asarray(cols, np.int64)
    o = np.lexsort((rows, cols))
    return np.searchsorted(cols[o], np.arange(sp + 1)), rows[o], rng.standard_normal((len(o), dn, dp))


def pairs(n0, n1, count, rng, must=()):
    """`count` distinct random (r, c) in an n0 x n1 grid, the pairs `must` among them"""
    must = np.asarray(list(must), np.int64).reshape(-1, 2)
    flat = np.unique(must[:, 0] * n1 + must[:, 1])
    while len(flat) < count:
        flat = np.union1d(flat, rng.integers(0, n0 * n1, 2 * (count - len(flat))))
    keep = np.isin(flat, must[:, 0] * n1 + must[:, 1])
    flat = np.concatenate([flat[keep], rng.permutation(flat[~keep])[:count - keep.sum()]])
    return flat // n1, flat % n1


def random_case(sm, sn, sp, dm, dn, dp, density, seed):
    rng = np.random.default_rng(seed)
    a = O.random_bsr(sm, sn, dm, dn, density, rng)
    ccol, row, v = O.transpose_pattern(*O.random_bsr(sp, sn, dp, dn, density, rng))
    return a, (ccol, row, np.ascontiguousarray(v)), sm, sn, sp


# ---------------------------------------------------------------------------------------------------------------------
# the three-way check
# ---------------------------------------------------------------------------------------------------------------------
def as_values(x, dtype, strided):
    """(nnz, d0, d1) values on the device, optionally as a view strided in every axis of a larger buffer"""
    t = torch.from_numpy(x).to(DEV, dtype)
    if not strided:
        return t
    n, d0, d1 = x.shape
    big = torch.full((2 * n, 2 * d0, 3 * d1), float("nan"), dtype=dtype, device=DEV)
    v = big[::2, 1::2, 2::3]
    v.copy_(t)
    assert not v.is_contiguous() and all(s != c for s, c in zip(v.stride(), t.stride()))
    return v


def same_bits(x, y):
    """bit for bit, the sign of zero included"""
    x, y = np.asarray(x), np.asarray(y)
    return x.dtype == y.dtype and x.shape == y.shape and np.array_equal(x.view(f"u{x.itemsize}"), y.view(f"u{y.itemsize}"))


def fwd_ptr(key):
    """segment pointers of the output blocks over the (i, j, k)-ordered triples"""
    return np.append(np.flatnonzero(np.r_[True, key[1:] != key[:-1]]), len(key)).astype(np.int64)


def host_grads(key, ta, tb, A, B, G):
    """dA and dB from the host build, replaying the regrouped triple orders exactly as bsr.cu grad_run does: dC is the
    left operand of dA and the right one of dB, B^T and A^T are read through swapped strides"""
    (nnz_a, dm, dn), (nnz_b, _, dp) = A.shape, B.shape
    tri, ptr = O.regroup(key, ta, tb, True, nnz_a)
    dA = host_numeric(G, [dm * dp, dp, 1], B, [dn * dp, 1, dp], tri, ptr, dm, dn, dp)
    tri, ptr = O.regroup(key, ta, tb, False, nnz_b)
    dB = host_numeric(A, [dm * dn, 1, dn], G, [dm * dp, dp, 1], tri, ptr, dn, dp, dm)
    return dA, dB


def bounded(got, want, mag, n, u):
    """-> the largest |got - want| / (gamma_n mag) (n per block).  Asserts the kernel is within gamma_n mag of the exact
    value, allowing the fp64 oracle its own gamma_{n+1}(2^-53) mag, and that a sum of no or only zero terms is +0.0."""
    got = np.asarray(got, np.float64)
    n = np.asarray(n, np.float64).reshape(-1, 1, 1)
    err = np.abs(got - want)
    bound = gamma(n, u) * mag
    bad = err > bound + gamma(n + 1, 2.0 ** -53) * mag
    assert not bad.any(), (err[bad][:5], bound[np.broadcast_to(bad, bound.shape)][:5] if bound.size else None)
    zero = mag == 0                                                   # no term, or only zero terms: exactly +0.0
    assert np.all(got[zero] == 0) and not np.signbit(got[zero]).any()
    return float((err[bound > 0] / bound[bound > 0]).max(initial=0.0))


def check(a, b, sm, sn, sp, dtype, *, seed=0, strided=False, ratios=None):
    """C = A B and both gradients on the device, checked three ways; -> {"fwd", "dA", "dB"} error / bound ratios."""
    npdt = np.float32 if dtype == F32 else np.float64
    u = np.finfo(npdt).eps / 2
    (a_crow, a_col, av), (b_ccol, b_row, bv) = a, b
    A, B = np.ascontiguousarray(av, npdt), np.ascontiguousarray(bv, npdt)   # what the device holds, read exactly in fp64
    (nnz_a, dm, dn), (nnz_b, _, dp) = A.shape, B.shape
    idx = [torch.from_numpy(np.asarray(x, np.int64)).to(DEV) for x in (a_crow, a_col, b_ccol, b_row)]
    va, vb = (as_values(x, dtype, strided).requires_grad_() for x in (A, B))
    out, crow, col = _BsrBscValues.apply(va, vb, *idx, sm, sn, sp)

    key, ta, tb = O.triples(a_crow, a_col, b_ccol, b_row, sp)
    c = O.blocks(key)
    wc, wl = O.pattern(a_crow, a_col, b_ccol, b_row, sm, sp)
    np.testing.assert_array_equal(crow.cpu().numpy(), wc)
    np.testing.assert_array_equal(col.cpu().numpy(), wl)
    _, _, tri, seg = out.grad_fn.saved_tensors
    want_tri = ((ta.astype(np.uint64) << np.uint64(32)) | tb.astype(np.uint64)).view(np.int64)
    assert np.array_equal(tri.cpu().numpy(), want_tri)                # the key sort's (i, j, k) order
    assert np.array_equal(seg.cpu().numpy(), c)

    got = out.detach().cpu().numpy()
    Ah, Bh = np.abs(A), np.abs(B)
    ptr = fwd_ptr(key)
    assert same_bits(got, host_numeric(A, [dm * dn, dn, 1], B, [dn * dp, dp, 1],
                                            (ta.astype(np.uint64) << np.uint64(32)) | tb.astype(np.uint64), ptr,
                                            dm, dp, dn))
    _, _, want = O.product(a_crow, a_col, A, b_ccol, b_row, B, sm, sp)
    _, _, mag = O.product(a_crow, a_col, Ah, b_ccol, b_row, Bh, sm, sp)
    r = {"fwd": bounded(got, want, mag, np.diff(ptr) * dn, u)}

    G = np.random.default_rng(seed + 1).standard_normal(got.shape).astype(npdt)
    ga, gb = torch.autograd.grad(out, (va, vb), torch.from_numpy(G).to(DEV))
    ga, gb = ga.cpu().numpy(), gb.cpu().numpy()
    hA, hB = host_grads(key, ta, tb, A, B, G)
    assert same_bits(ga, hA) and same_bits(gb, hB)
    wA, wB = O.grads(a_crow, a_col, A, b_ccol, b_row, B, sm, sp, G)
    mA, mB = O.grads(a_crow, a_col, Ah, b_ccol, b_row, Bh, sm, sp, np.abs(G))
    r["dA"] = bounded(ga, wA, mA, np.bincount(ta, minlength=nnz_a) * dp, u)
    r["dB"] = bounded(gb, wB, mB, np.bincount(tb, minlength=nnz_b) * dm, u)
    if ratios is not None:
        ratios(str(dtype)[6:], r)
    return r


@pytest.fixture
def ratios(record_property):
    def rec(dt, r):
        record_property(f"ratio_{dt}", r)
        print(f"ratio {dt} " + " ".join(f"{k}={v:.3g}" for k, v in r.items()))
    return rec


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the oracle's gradients and triple orders, the host replay, the width mirror
# ---------------------------------------------------------------------------------------------------------------------
SHAPES = [(7, 6, 5, 2, 3, 4), (5, 8, 6, 3, 1, 2), (6, 4, 7, 1, 5, 1), (4, 9, 3, 5, 2, 3)]


def dense_case(sm, sn, sp, dm, dn, dp, seed):
    """a random case with an empty A row, an empty B column and stored zero blocks in both operands"""
    a, b, *_ = random_case(sm, sn, sp, dm, dn, dp, 0.5, seed)
    (a_crow, a_col, av), (b_ccol, b_row, bv) = a, b
    drop = np.arange(a_crow[1], a_crow[2])                            # A row 1 and B column 2 emptied
    a = (a_crow - np.clip(np.arange(sm + 1) - 1, 0, 1) * len(drop), np.delete(a_col, drop), np.delete(av, drop, 0))
    drop = np.arange(b_ccol[2], b_ccol[3])
    b = (b_ccol - np.clip(np.arange(sp + 1) - 2, 0, 1) * len(drop), np.delete(b_row, drop), np.delete(bv, drop, 0))
    a[2][::3], b[2][::4] = 0.0, 0.0
    return a, b


def dense(crow, col, val, size, layout):
    f = torch.sparse_bsr_tensor if layout == "bsr" else torch.sparse_bsc_tensor
    return f(torch.from_numpy(crow), torch.from_numpy(col), torch.from_numpy(np.ascontiguousarray(val)), size=size).to_dense()


def blocks_of(D, crow, col, dm, dn, bsc_=False):
    """the stored blocks of a dense matrix in BSR (or BSC) order"""
    seg = np.repeat(np.arange(len(crow) - 1), np.diff(crow))
    r, c = (col, seg) if bsc_ else (seg, col)
    return np.stack([D[i * dm:(i + 1) * dm, j * dn:(j + 1) * dn] for i, j in zip(r, c)]) if len(col) else \
        np.zeros((0, dm, dn))


@pytest.mark.parametrize("shape", SHAPES)
def test_grads_match_dense_autograd(shape):
    sm, sn, sp, dm, dn, dp = shape
    a, b = dense_case(*shape, seed=sum(shape))
    assert np.diff(a[0])[1] == 0 and np.diff(b[0])[2] == 0 and (a[2] == 0).all((1, 2)).any()
    Ad = dense(*a, (sm * dm, sn * dn), "bsr").requires_grad_()
    Bd = dense(*b, (sn * dn, sp * dp), "bsc").requires_grad_()
    crow, col = O.pattern(a[0], a[1], b[0], b[1], sm, sp)
    G = np.random.default_rng(1).standard_normal((len(col), dm, dp))
    W = dense(crow, col, G, (sm * dm, sp * dp), "bsr")
    gA, gB = torch.autograd.grad((W * (Ad @ Bd)).sum(), (Ad, Bd))
    dA, dB = O.grads(*a, *b, sm, sp, G)
    np.testing.assert_allclose(dA, blocks_of(gA.numpy(), a[0], a[1], dm, dn), rtol=0, atol=1e-12)
    np.testing.assert_allclose(dB, blocks_of(gB.numpy(), b[0], b[1], dn, dp, bsc_=True), rtol=0, atol=1e-12)


@pytest.mark.parametrize("shape", SHAPES[:2])
def test_grads_of_a_at(shape):
    sm, sn, _, dm, dn, _ = shape
    a, _ = dense_case(*shape, seed=7)
    Ad = dense(*a, (sm * dm, sn * dn), "bsr").requires_grad_()
    crow, col = O.pattern(a[0], a[1], a[0], a[1], sm, sm)
    G = np.random.default_rng(2).standard_normal((len(col), dm, dm))
    W = dense(crow, col, G, (sm * dm, sm * dm), "bsr")
    (gA,) = torch.autograd.grad((W * (Ad @ Ad.mT)).sum(), (Ad,))
    dA, dB = O.grads(*a, *O.transpose_pattern(*a), sm, sm, G)
    np.testing.assert_allclose(dA + dB.swapaxes(1, 2), blocks_of(gA.numpy(), a[0], a[1], dm, dn), rtol=0, atol=1e-12)


@pytest.mark.parametrize("shape", SHAPES)
def test_host_replay_of_the_regrouped_triples(shape):
    sm, _, sp, dm, _, dp = shape
    a, b = dense_case(*shape, seed=3)
    key, ta, tb = O.triples(a[0], a[1], b[0], b[1], sp)
    G = np.random.default_rng(4).standard_normal((len(np.unique(key)), dm, dp))
    hA, hB = host_grads(key, ta, tb, np.ascontiguousarray(a[2]), np.ascontiguousarray(b[2]), G)
    wA, wB = O.grads(*a, *b, sm, sp, G)
    np.testing.assert_allclose(hA, wA, rtol=0, atol=1e-12)
    np.testing.assert_allclose(hB, wB, rtol=0, atol=1e-12)
    tri, ptr = O.regroup(key, ta, tb, True, len(a[1]))
    assert np.array_equal(np.diff(ptr), np.bincount(ta, minlength=len(a[1])))
    assert np.all(np.diff((tri >> np.uint64(32)).astype(np.int64)[ptr[0]:ptr[1]]) >= 0)   # c ascending within an entry


def test_bits_of_at_the_boundaries():
    for v, w in [(0, 1), (1, 1), (2, 2), (3, 2), (4, 3), (2 ** 16 - 1, 16), (2 ** 16, 17), (2 ** 17 - 1, 17),
                 (2 ** 17, 18), (2 ** 32 - 1, 32), (2 ** 32, 33), (2 ** 63, 64), (2 ** 64 - 1, 64)]:
        assert bits_of(v) == w, v
    assert widths(1, 1, 1, 1, 1) == {"brow": 1, "key": 1, "dA": 1, "dB": 1}
    assert widths(64, 2 ** 17, 64, 2, 2)["brow"] == 17 and widths(64, 2 ** 17 + 1, 64, 2, 2)["brow"] == 18
    assert widths(2 ** 16, 32, 2 ** 16, 2, 2)["key"] == 32 and widths(2 ** 16 + 1, 32, 2 ** 16, 2, 2)["key"] == 33
    assert widths(32, 4096, 32, 2 ** 16, 2 ** 16)["dA"] == 16 and widths(32, 4096, 32, 2 ** 16 + 1, 2 ** 16 + 1)["dB"] == 17


def test_regroup_orders_are_stable():
    key = np.array([0, 0, 1, 3, 3, 3])
    a, b = np.array([2, 0, 2, 1, 2, 0]), np.array([1, 0, 0, 1, 0, 2])
    tri, ptr = O.regroup(key, a, b, True, 4)
    c = O.blocks(key)
    assert c.tolist() == [0, 0, 1, 2, 2, 2] and ptr.tolist() == [0, 2, 3, 6, 6]
    assert tri.tolist() == [(0 << 32) | 0, (2 << 32) | 2, (2 << 32) | 1, (0 << 32) | 1, (1 << 32) | 0, (2 << 32) | 0]
    tri, ptr = O.regroup(key, a, b, False, 3)
    assert ptr.tolist() == [0, 3, 5, 6]
    assert tri.tolist() == [(0 << 32) | 0, (2 << 32) | 1, (2 << 32) | 2, (2 << 32) | 0, (1 << 32) | 2, (0 << 32) | 2]


# ---------------------------------------------------------------------------------------------------------------------
# GPU: sort widths at their boundaries
# ---------------------------------------------------------------------------------------------------------------------
def interleaved(keys, w):
    """keys on both sides of bit w - 1, one with it set before one without"""
    top = (np.asarray(keys, np.int64) >> (w - 1)) & 1
    return bool(np.any(np.diff(top) < 0))


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [F32, F64])
@pytest.mark.parametrize("sn,w", [(2 ** 17, 17), (2 ** 17 + 1, 18)])
def test_b_row_sort_width(sn, w, dtype, ratios):
    """every B column holds rows on both sides of the top bit, the last row sn - 1 among them"""
    rng = np.random.default_rng(sn)
    sm = sp = 48
    pool = np.unique(np.concatenate([[0, 1, 2 ** 16 - 1, 2 ** 16, sn - 2, sn - 1], rng.integers(0, sn, 60)]))
    ar, ac = pairs(sm, len(pool), 600, rng, must=[(i, len(pool) - 1) for i in range(0, sm, 3)])
    a = bsr(ar, pool[ac], sm, 2, 3, rng)
    br, bc = pairs(len(pool), sp, 800, rng, must=[(len(pool) - 1, j) for j in range(sp)] + [(0, j) for j in range(sp)])
    b = bsc(pool[br], bc, sp, 3, 2, rng)
    assert widths(sm, sn, sp, len(a[1]), len(b[1]))["brow"] == w
    assert b[1].max() == sn - 1 and interleaved(b[1], w)
    check(a, b, sm, sn, sp, dtype, seed=sn, ratios=ratios)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [F32, F64])
@pytest.mark.parametrize("sm,sp,w", [(2 ** 16, 2 ** 16, 32), (2 ** 16 + 1, 2 ** 16, 33)])
def test_key_sort_width(sm, sp, w, dtype, ratios):
    """products in the first and the last block row and column, and on both sides of the key's top bit"""
    rng = np.random.default_rng(sm)
    sn = 32
    rows = np.unique(np.concatenate([[0, 1, 2 ** 15 - 1, 2 ** 15, sm - 2, sm - 1], rng.integers(0, sm, 300)]))
    cols = np.unique(np.concatenate([[0, 1, 2 ** 15, sp - 1], rng.integers(0, sp, 300)]))
    ar, ac = pairs(len(rows), sn, 5 * len(rows), rng, must=[(0, 0), (len(rows) - 1, 0)])
    a = bsr(rows[ar], ac, sm, 3, 2, rng)
    br, bc = pairs(sn, len(cols), 5 * len(cols), rng, must=[(0, 0), (0, len(cols) - 1)])
    b = bsc(br, cols[bc], sp, 2, 3, rng)
    assert widths(sm, sn, sp, len(a[1]), len(b[1]))["key"] == w
    key, _, _ = O.triples(*a[:2], *b[:2], sp)
    assert key.min() == 0 and key.max() == sm * sp - 1 and (key >> (w - 1)).any() and not (key >> (w - 1)).all()
    check(a, b, sm, sn, sp, dtype, seed=sm, ratios=ratios)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [F32, F64])
@pytest.mark.parametrize("nnz,w", [(2 ** 16, 16), (2 ** 16 + 1, 17)])
def test_regroup_sort_widths(nnz, w, dtype, ratios):
    """nnzA = nnzB = nnz, about 2^20 block products, each regroup's keys on both sides of its top bit interleaved in the
    (i, j, k) order"""
    rng = np.random.default_rng(nnz)
    sm, sn, sp = 32, 4096, 32
    a = bsr(*pairs(sm, sn, nnz, rng, must=[(sm - 1, k) for k in range(0, sn, 512)]), sm, 2, 3, rng)
    br, bc = pairs(sn, sp, nnz, rng, must=[(k, sp - 1) for k in range(0, sn, 512)])
    b = bsc(br, bc, sp, 3, 2, rng)
    assert widths(sm, sn, sp, nnz, nnz)["dA"] == w and widths(sm, sn, sp, nnz, nnz)["dB"] == w
    _, ta, tb = O.triples(*a[:2], *b[:2], sp)
    assert interleaved(ta, w) and interleaved(tb, w) and ta.max() == tb.max() == nnz - 1
    check(a, b, sm, sn, sp, dtype, seed=nnz, ratios=ratios)


def _degenerate(name):
    rng = np.random.default_rng(len(name))
    if name == "all_one":
        return bsr([0], [0], 1, 2, 3, rng), bsc([0], [0], 1, 3, 2, rng), 1, 1, 1
    if name == "sm1":
        return bsr(np.zeros(20, int), rng.permutation(50)[:20], 1, 2, 3, rng), bsc(*pairs(50, 30, 400, rng), 30, 3, 2, rng), \
            1, 50, 30
    if name == "sp1":
        return bsr(*pairs(30, 50, 400, rng), 30, 2, 3, rng), bsc(rng.permutation(50)[:20], np.zeros(20, int), 1, 3, 2, rng), \
            30, 50, 1
    if name == "sn1":
        return bsr(np.arange(0, 30, 2), np.zeros(15, int), 30, 2, 3, rng), bsc(np.zeros(12, int), np.arange(1, 25, 2), 25, 3,
                                                                                 2, rng), 30, 1, 25
    if name == "nnzA1":
        return bsr([3], [7], 10, 2, 3, rng), bsc(*pairs(20, 15, 120, rng, must=[(7, 0), (7, 14)]), 15, 3, 2, rng), \
            10, 20, 15
    if name == "nnzB1":
        return bsr(*pairs(10, 20, 80, rng, must=[(0, 7), (9, 7)]), 10, 2, 3, rng), bsc([7], [4], 15, 3, 2, rng), \
            10, 20, 15


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [F32, F64])
@pytest.mark.parametrize("name,one", [("all_one", ("brow", "key", "dA", "dB")), ("sm1", ()), ("sp1", ()),
                                      ("sn1", ("brow",)), ("nnzA1", ("dA",)), ("nnzB1", ("dB",))])
def test_degenerate_sizes(name, one, dtype, ratios):
    """sm, sp, sn, nnzA or nnzB of one: bits_of(0) = 1 sorts"""
    a, b, sm, sn, sp = _degenerate(name)
    w = widths(sm, sn, sp, len(a[1]), len(b[1]))
    assert all(w[k] == 1 for k in one)
    if name in ("sm1", "sp1"):
        assert w["key"] == bits_of(max(sm, sp) - 1)
    check(a, b, sm, sn, sp, dtype, seed=3, ratios=ratios)


# ---------------------------------------------------------------------------------------------------------------------
# GPU: block shapes, long segments, structural zeros, strides and index dtypes
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [F32, F64])
@pytest.mark.parametrize("blk", [(1, 1, 1), (1, 32, 1), (16, 1, 16), (3, 5, 7), (7, 3, 5), (8, 8, 8), (32, 32, 32)],
                         ids=lambda b: "x".join(map(str, b)))
def test_block_shapes(blk, dtype, ratios):
    check(*random_case(20, 16, 18, *blk, 0.25, seed=sum(blk)), dtype, seed=sum(blk), ratios=ratios)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [F32, F64])
def test_long_segments(dtype, ratios):
    """a dense block row of A across a dense block column of B over sn = 4096: one output block sums 4096 dz terms"""
    rng = np.random.default_rng(5)
    sm, sn, sp = 4, 4096, 4
    ar, ac = pairs(sm, sn, 4096 + 400, rng, must=[(1, k) for k in range(sn)])
    br, bc = pairs(sn, sp, 4096 + 400, rng, must=[(k, 2) for k in range(sn)])
    a, b = bsr(ar, ac, sm, 2, 4, rng), bsc(br, bc, sp, 4, 2, rng)
    key, _, _ = O.triples(*a[:2], *b[:2], sp)
    assert np.diff(fwd_ptr(key)).max() * 4 == 4096 * 4
    check(a, b, sm, sn, sp, dtype, seed=5, ratios=ratios)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [F32, F64])
def test_permutation_product(dtype, ratios):
    """block-diagonal A times a permuted block-diagonal B: one product per output block, and the output block c of a
    product differs from its B entry b, so a triple packed with c and b swapped reads other blocks"""
    rng = np.random.default_rng(14)
    n = 300
    perm = rng.permutation(n)
    a, b = bsr(np.arange(n), np.arange(n), n, 3, 2, rng), bsc(perm, np.arange(n), n, 2, 4, rng)
    key, ta, tb = O.triples(*a[:2], *b[:2], n)
    assert len(key) == n and (O.blocks(key) != tb).mean() > 0.9
    check(a, b, n, n, n, dtype, seed=14, ratios=ratios)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [F32, F64])
def test_structural_zeros(dtype, ratios):
    """A entries without a partner in B, B entries never used, an empty A row and B column, and stored zero blocks: the
    gradients of the unpartnered entries are exactly +0.0 and zero blocks still form output blocks (check())"""
    rng = np.random.default_rng(6)
    sm, sn, sp = 10, 12, 9
    ar, ac = pairs(sm, sn, 50, rng, must=[(0, 7), (4, 7), (2, 1), (2, 2)])
    keep = (ar != 3) & ~np.isin(ac, [9])                              # A row 3 empty, nothing in A's column 9
    br, bc = pairs(sn, sp, 50, rng, must=[(9, 0), (9, 4), (1, 6), (2, 6)])
    kb = (bc != 5) & (br != 7)                                        # B column 5 empty, nothing in B's row 7
    a, b = bsr(ar[keep], ac[keep], sm, 2, 3, rng), bsc(br[kb], bc[kb], sp, 3, 4, rng)
    a[2][a[0][2]:a[0][3]] = 0.0                                      # C's block row 2 sums zero blocks only
    a[2][::5], b[2][::6] = 0.0, 0.0
    key, ta, tb = O.triples(*a[:2], *b[:2], sp)
    assert np.diff(a[0])[3] == 0 and np.diff(b[0])[5] == 0 and 2 * sp + 6 in key
    assert (np.bincount(ta, minlength=len(a[1])) == 0).any() and (np.bincount(tb, minlength=len(b[1])) == 0).any()
    check(a, b, sm, sn, sp, dtype, seed=6, ratios=ratios)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [F32, F64])
@pytest.mark.parametrize("blk", [(3, 5, 7), (7, 3, 5)], ids=lambda b: "x".join(map(str, b)))
def test_strided_values(blk, dtype, ratios):
    """both operands' values strided in every axis, in the forward and both gradients"""
    check(*random_case(20, 16, 18, *blk, 0.25, seed=9), dtype, seed=9, strided=True, ratios=ratios)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [F32, F64])
@pytest.mark.parametrize("idx", [torch.int32, torch.int64])
def test_index_dtypes_through_the_sparse_constructors(idx, dtype):
    """pp.bsr_bsc_matmul on int32 / int64 indices and strided values, gradients through torch.sparse_bsr_tensor /
    .values(): bit for bit the values-level results"""
    (a_crow, a_col, av), (b_ccol, b_row, bv), sm, sn, sp = random_case(9, 7, 8, 3, 2, 4, 0.35, seed=10)
    va, vb = as_values(av, dtype, True).requires_grad_(), as_values(bv, dtype, True).requires_grad_()
    ti = lambda x: torch.from_numpy(x).to(DEV, idx)   # noqa: E731
    A = torch.sparse_bsr_tensor(ti(a_crow), ti(a_col), va, size=(sm * 3, sn * 2))
    B = torch.sparse_bsc_tensor(ti(b_ccol), ti(b_row), vb, size=(sn * 2, sp * 4))
    assert A.crow_indices().dtype == idx and not A.values().is_contiguous() and not B.values().is_contiguous()
    C = pp.bsr_bsc_matmul(A, B)
    W = torch.randn_like(C.values())
    ga, gb = torch.autograd.grad((C.values() * W).sum(), (va, vb))
    l64 = lambda x: torch.from_numpy(x).to(DEV)       # noqa: E731
    out, crow, col = _BsrBscValues.apply(va, vb, l64(a_crow), l64(a_col), l64(b_ccol), l64(b_row), sm, sn, sp)
    wa, wb = torch.autograd.grad(out, (va, vb), W)
    assert torch.equal(C.crow_indices(), crow) and torch.equal(C.col_indices(), col)
    assert torch.equal(C.values(), out) and torch.equal(ga, wa) and torch.equal(gb, wb)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [F32, F64])
def test_requires_grad_subsets(dtype):
    """{A}, {B} and {A, B}: each requested gradient bit-identical"""
    a, b, sm, sn, sp = random_case(12, 10, 11, 3, 5, 2, 0.3, seed=11)
    idx = [torch.from_numpy(x).to(DEV) for x in (a[0], a[1], b[0], b[1])]
    va0, vb0 = as_values(a[2], dtype, False), as_values(b[2], dtype, False)
    W = torch.randn(len(O.pattern(a[0], a[1], b[0], b[1], sm, sp)[1]), 3, 2, dtype=dtype, device=DEV)
    got = {}
    for req in ("A", "B", "AB"):
        va, vb = va0.clone().requires_grad_("A" in req), vb0.clone().requires_grad_("B" in req)
        out, _, _ = _BsrBscValues.apply(va, vb, *idx, sm, sn, sp)
        ins = [v for v, r in ((va, "A"), (vb, "B")) if r in req]
        got[req] = dict(zip([r for r in "AB" if r in req], torch.autograd.grad(out, ins, W)))
    assert torch.equal(got["A"]["A"], got["AB"]["A"]) and torch.equal(got["B"]["B"], got["AB"]["B"])


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [F32, F64])
def test_a_at_shared_path(dtype):
    """A @ A.mT passes A's values once: its gradient is bit for bit dA + dB^T of the non-shared call on a contiguous copy
    of A^T"""
    crow, col, val = O.random_bsr(40, 30, 3, 5, 0.15, np.random.default_rng(12))
    ct, lt = torch.from_numpy(crow).to(DEV), torch.from_numpy(col).to(DEV)
    va = torch.from_numpy(val).to(DEV, dtype).requires_grad_()
    out = values_product(va, None, ct, lt, ct, lt, 40, 30, 40)
    W = torch.randn_like(out)
    (g,) = torch.autograd.grad(out, va, W)
    vb = va.detach().mT.contiguous().requires_grad_()
    out2 = values_product(va, vb, ct, lt, ct, lt, 40, 30, 40)
    ga, gb = torch.autograd.grad(out2, (va, vb), W)
    assert torch.equal(out, out2) and torch.equal(g, ga + gb.mT)


# ---------------------------------------------------------------------------------------------------------------------
# GPU: scale, reproducibility, the second grid-stride pass, the product cap
# ---------------------------------------------------------------------------------------------------------------------
def pattern_1e5(n=100000, per=10, seed=11):
    """tests/test_sparse.py's 1e5 x 1e5 grid, 10 blocks per row from 64 reused row patterns: about 1e7 block products
    of A A^T"""
    rng = np.random.default_rng(seed)
    col = np.sort(np.stack([rng.choice(n, per, replace=False) for _ in range(64)]), 1)
    col = np.sort((col[rng.integers(0, 64, n)] + rng.integers(0, n, (n, 1))) % n, 1)
    keep = np.concatenate([np.ones((n, 1), bool), np.diff(col, axis=1) > 0], 1)
    crow = np.concatenate([[0], np.cumsum(keep.sum(1))]).astype(np.int64)
    return crow, col[keep].astype(np.int64), rng.standard_normal((int(keep.sum()), 2, 2)), rng


def rows_of(crow, col, val, S):
    """the entries of the block rows S (sorted) of a BSR matrix, every other row emptied -> ((crow, col, val), entries);
    the same for the block columns S of a BSC matrix"""
    ents = np.concatenate([np.arange(crow[r], crow[r + 1]) for r in S])
    cnt = np.zeros(len(crow) - 1, np.int64)
    cnt[S] = np.diff(crow)[S]
    return (np.concatenate([[0], np.cumsum(cnt)]), col[ents], np.ascontiguousarray(val[ents])), ents


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [F32, F64])
def test_a_at_1e5_block_rows(dtype, ratios):
    """the gradient of A @ A.mT at about 1e7 block products (CUB's multi-pass radix sorts), on 200 block rows against
    the oracle and the host build; bit-identical over two runs and on a side stream"""
    n = 100000
    crow, col, val, rng = pattern_1e5(n)
    npdt = np.float32 if dtype == F32 else np.float64
    A = val.astype(npdt)
    Bt = np.ascontiguousarray(A.swapaxes(1, 2))                       # B = A^T in BSC: A's pattern, transposed blocks
    assert (np.bincount(col, minlength=n) ** 2).sum() > 8e6         # block products: sum over k of |A's column k|^2
    assert widths(n, n, n, len(col), len(col)) == {"brow": 17, "key": 34, "dA": bits_of(len(col) - 1),
                                                   "dB": bits_of(len(col) - 1)}
    ct, lt = torch.from_numpy(crow).to(DEV), torch.from_numpy(col).to(DEV)
    va = torch.from_numpy(A).to(DEV).requires_grad_()

    def run():
        out, c_crow, c_col = _BsrBscValues.apply(va, None, ct, lt, ct, lt, n, n, n)
        return out.detach(), torch.autograd.grad(out, va, W)[0], c_crow, c_col
    n_c = _BsrBscValues.apply(va.detach(), None, ct, lt, ct, lt, n, n, n)[0].shape[0]
    W = torch.from_numpy(np.random.default_rng(1).standard_normal((n_c, 2, 2)).astype(npdt)).to(DEV)
    out, g, c_crow, c_col = run()
    out2, g2, _, _ = run()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        out3, g3, _, _ = run()
    torch.cuda.current_stream().wait_stream(side)
    assert torch.equal(out, out2) and torch.equal(g, g2) and torch.equal(out, out3) and torch.equal(g, g3)

    # dA of the entries in rows S needs only the products of A's rows S; dB of the same entries (B's columns S) only
    # the products with B's columns S.  Each is a small product whose triples keep the full product's relative order.
    G, got = W.cpu().numpy(), g.cpu().numpy()
    c_crow, c_col = c_crow.cpu().numpy(), c_col.cpu().numpy()
    S = np.sort(rng.choice(n, 200, replace=False))
    a_s, ents = rows_of(crow, col, A, S)
    b_s, _ = rows_of(crow, col, Bt, S)
    G_rows = G[np.concatenate([np.arange(c_crow[r], c_crow[r + 1]) for r in S])]
    G_cols = G[np.isin(c_col, S)]
    key, ta, tb = O.triples(*a_s[:2], crow, col, n)
    tri, ptr = O.regroup(key, ta, tb, True, len(ents))
    hA = host_numeric(G_rows, [4, 2, 1], Bt, [4, 1, 2], tri, ptr, 2, 2, 2)
    nA = np.bincount(ta, minlength=len(ents))
    key, ta, tb = O.triples(crow, col, *b_s[:2], n)
    tri, ptr = O.regroup(key, ta, tb, False, len(ents))
    hB = host_numeric(A, [4, 1, 2], G_cols, [4, 2, 1], tri, ptr, 2, 2, 2)
    nB = np.bincount(tb, minlength=len(ents))
    assert same_bits(got[ents], hA + hB.swapaxes(1, 2))
    wA, _ = O.grads(*a_s, crow, col, Bt, n, n, G_rows)
    mA, _ = O.grads(*a_s[:2], np.abs(a_s[2]), crow, col, np.abs(Bt), n, n, np.abs(G_rows))
    _, wB = O.grads(crow, col, A, *b_s, n, n, G_cols)
    _, mB = O.grads(crow, col, np.abs(A), *b_s[:2], np.abs(b_s[2]), n, n, np.abs(G_cols))
    # the shared gradient adds the two chains: within the bound of one chain of their total length plus one
    r = {"dA+dB^T": bounded(got[ents], wA + wB.swapaxes(1, 2), mA + mB.swapaxes(1, 2), (nA + nB) * 2 + 1, np.finfo(npdt).eps / 2)}
    ratios(str(dtype)[6:], r)


def _block_diagonal_fp32(N, d, sel):
    """C = A B and both gradients of a block-diagonal fp32 product of N (d x d) blocks on the device -> the blocks sel of
    A, B, dC, C, dA and dB on the host, whether the pattern is the diagonal, and the peak device memory it took.  The
    device memory is freed when it returns."""
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    gen = torch.Generator(device=DEV).manual_seed(13)
    ar = torch.arange(N + 1, dtype=torch.int64, device=DEV)
    va = torch.randn(N, d, d, generator=gen, device=DEV).requires_grad_()
    vb = torch.randn(N, d, d, generator=gen, device=DEV).requires_grad_()
    W = torch.randn(N, d, d, generator=gen, device=DEV)
    out, crow, col = _BsrBscValues.apply(va, vb, ar, ar[:-1], ar, ar[:-1], N, N, N)
    diagonal = torch.equal(crow, ar) and torch.equal(col, ar[:-1]) and out.shape == (N, d, d)
    ga, gb = torch.autograd.grad(out, (va, vb), W)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    idx = torch.from_numpy(sel).to(DEV)
    host = [x.detach()[idx].cpu().numpy() for x in (va, vb, W, out, ga, gb)]
    del va, vb, W, out, crow, col, ga, gb, ar, idx
    torch.cuda.empty_cache()
    return host, diagonal, peak


@pytest.mark.gpu
def test_second_grid_stride_pass(record_property):
    """fp32 block-diagonal product of 2^20 + 4099 (16 x 16) blocks: the forward and both gradients have more than 2^28
    elements, so one grid-stride pass of the numeric kernel does not cover them.  Every element past 2^28 and a random
    sample of the rest against the host build."""
    N, d = (1 << 20) + 4099, 16
    assert N * d * d > PASS and N - PASS // (d * d) == 4099
    rng = np.random.default_rng(13)
    sel = np.concatenate([np.sort(rng.choice(PASS // (d * d), 2000, replace=False)), np.arange(PASS // (d * d), N)])
    (A, B, G, C, dA, dB), diagonal, peak = _block_diagonal_fp32(N, d, sel)
    record_property("peak_bytes", peak)
    print(f"peak device memory {peak / 2 ** 30:.2f} GiB")
    assert diagonal
    m = len(sel)
    one = (np.arange(m, dtype=np.uint64) << np.uint64(32)) | np.arange(m, dtype=np.uint64)   # triple (c, c) of block c
    ptr = np.arange(m + 1, dtype=np.int64)
    s, t = [d * d, d, 1], [d * d, 1, d]
    assert same_bits(C, host_numeric(A, s, B, s, one, ptr, d, d, d))
    assert same_bits(dA, host_numeric(G, s, B, t, one, ptr, d, d, d))
    assert same_bits(dB, host_numeric(A, t, G, s, one, ptr, d, d, d))


@pytest.mark.gpu
def test_product_cap_raises_after_the_count(monkeypatch):
    """1 x 1 blocks, sm = sp = 2048 over a dense sn = 513: 2048 * 513 * 2048 > 2^31 - 1 block products"""
    sm, sn, sp = 2048, 513, 2048
    assert sm * sn * sp > INT31
    ar = torch.arange(sm + 1, dtype=torch.int64, device=DEV) * sn
    ks = torch.arange(sn, dtype=torch.int64, device=DEV).repeat(sm)
    va = torch.ones(sm * sn, 1, 1, dtype=F32, device=DEV)
    called, fn = [], _C.fn
    monkeypatch.setattr(_C, "fn", lambda s: called.append(s) or fn(s))
    with pytest.raises(ValueError, match="exceed"):
        _BsrBscValues.apply(va, va.clone(), ar, ks, ar, ks, sm, sn, sp)
    assert called == ["b200_bsr_count"]
