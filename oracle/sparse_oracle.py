"""numpy oracle of pp.bsr_bsc_matmul (csrc/bsr.cu): the structural output pattern of a BSR × BSC product and its fp64
values, the fp64 gradients of both values arrays, and the triple orders the kernels accumulate in.  Used for the cases
the reference is too slow for, and checked against the reference's goldens (tests/golden/sparse.npz,
oracle/make_golden_sparse.py).

A is given as (crow, col, values (nnzA, dm, dn)), B as (ccol, row, values (nnzB, dn, dp)).  Block (i, j) of C exists
exactly when block row i of A and block column j of B share a stored block index k, stored zero blocks included.
"""
import numpy as np


def triples(a_crow, a_col, b_ccol, b_row, sp):
    """(key = i * sp + j, a, b) of every block product, sorted by (i, j, k)."""
    a_crow, a_col = np.asarray(a_crow, np.int64), np.asarray(a_col, np.int64)
    b_ccol, b_row = np.asarray(b_ccol, np.int64), np.asarray(b_row, np.int64)
    nnz_a, nnz_b = len(a_col), len(b_row)
    a_i = np.repeat(np.arange(len(a_crow) - 1), np.diff(a_crow))
    b_j = np.repeat(np.arange(len(b_ccol) - 1), np.diff(b_ccol))
    bt = np.argsort(b_row, kind="stable")                 # B's entries by row, by column within a row
    sn = int(max(a_col.max(initial=-1), b_row.max(initial=-1))) + 1
    bt_ptr = np.searchsorted(b_row[bt], np.arange(sn + 1))
    cnt = bt_ptr[a_col + 1] - bt_ptr[a_col] if nnz_a and nnz_b else np.zeros(nnz_a, np.int64)
    a = np.repeat(np.arange(nnz_a), cnt)
    start = np.repeat(np.cumsum(cnt) - cnt, cnt)
    b = bt[bt_ptr[a_col[a]] + np.arange(len(a)) - start] if len(a) else np.zeros(0, np.int64)
    key = a_i[a] * sp + b_j[b]
    o = np.lexsort((a_col[a], key))
    return key[o], a[o], b[o]


def pattern(a_crow, a_col, b_ccol, b_row, sm, sp):
    """crow (sm + 1) and col of C, int64."""
    key, _, _ = triples(a_crow, a_col, b_ccol, b_row, sp)
    u = np.unique(key)
    crow = np.searchsorted(u, np.arange(sm + 1) * sp).astype(np.int64)
    return crow, (u % sp).astype(np.int64)


def product(a_crow, a_col, a_val, b_ccol, b_row, b_val, sm, sp, rows=None):
    """crow, col and fp64 values of C.  With `rows` (sorted block rows), only those rows' values are formed: the returned
    values then cover the output blocks crow[r] .. crow[r + 1] - 1 of each r, in order."""
    key, a, b = triples(a_crow, a_col, b_ccol, b_row, sp)
    u, seg = np.unique(key, return_inverse=True)
    crow = np.searchsorted(u, np.arange(sm + 1) * sp).astype(np.int64)
    col = (u % sp).astype(np.int64)
    A, B = np.asarray(a_val, np.float64), np.asarray(b_val, np.float64)
    if rows is not None:
        keep = np.isin(key // sp, np.asarray(rows))
        a, b, seg = a[keep], b[keep], seg[keep]
        blocks = np.concatenate([np.arange(crow[r], crow[r + 1]) for r in rows]) if len(rows) else np.zeros(0, np.int64)
        seg = np.searchsorted(blocks, seg)
        n = len(blocks)
    else:
        n = len(u)
    out = np.zeros((n, A.shape[1], B.shape[2]))
    np.add.at(out, seg, np.einsum("tij,tjk->tik", A[a], B[b]))
    return crow, col, out


def grads(a_crow, a_col, a_val, b_ccol, b_row, b_val, sm, sp, dC):
    """fp64 dA (nnzA, dm, dn) and dB (nnzB, dn, dp) of <dC, C> for dC (nnz(C), dm, dp) in C's block order:
    dA[a] += dC[c] B[b]^T and dB[b] += A[a]^T dC[c] over every block product (c, a, b)."""
    key, a, b = triples(a_crow, a_col, b_ccol, b_row, sp)
    c = blocks(key)
    A, B, G = (np.asarray(x, np.float64) for x in (a_val, b_val, dC))
    dA, dB = np.zeros(A.shape), np.zeros(B.shape)
    np.add.at(dA, a, np.einsum("tik,tjk->tij", G[c], B[b]))
    np.add.at(dB, b, np.einsum("tji,tjk->tik", A[a], G[c]))
    return dA, dB


def regroup(key, a, b, by_a, n):
    """The gradient kernels' triple order (csrc/bsr.cu grad_run): the (i, j, k)-ordered triples of `triples()` sorted
    stably by a (by_a) or by b, packed as (c << 32) | b or (a << 32) | c.  -> (tri uint64, ptr (n + 1) int64), where
    entry e of the n entries of A (by_a) or B sums the triples ptr[e] .. ptr[e + 1] - 1."""
    c = blocks(key)
    g = np.asarray(a if by_a else b, np.int64)
    hi, lo = (c, b) if by_a else (a, c)
    o = np.argsort(g, kind="stable")
    tri = (np.asarray(hi, np.uint64)[o] << np.uint64(32)) | np.asarray(lo, np.uint64)[o]
    return tri, np.searchsorted(g[o], np.arange(n + 1)).astype(np.int64)


def blocks(key):
    """output block c of every triple, for keys in (i, j, k) order"""
    return np.concatenate([[0], np.cumsum(key[1:] != key[:-1])]).astype(np.int64) if len(key) else \
        np.zeros(0, np.int64)


def random_bsr(sm, sn, dm, dn, density, rng, zero_prob=0.0, dtype=np.float64):
    """(crow, col, values) of a random BSR pattern: each block present with probability `density`."""
    mask = rng.random((sm, sn)) < density
    crow = np.concatenate([[0], np.cumsum(mask.sum(1))]).astype(np.int64)
    col = np.nonzero(mask)[1].astype(np.int64)
    val = rng.standard_normal((len(col), dm, dn))
    val[rng.random(val.shape) < zero_prob] = 0.0
    return crow, col, val.astype(dtype)


def transpose_pattern(crow, col, val):
    """The BSC (ccol, row, values) of the transpose of a BSR matrix: B = A^T has ccol = crow, row = col, values^T."""
    return crow, col, np.swapaxes(val, 1, 2)
