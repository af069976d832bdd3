"""Goldens for pp.bsr_bsc_matmul from the REFERENCE (pypose v0.9.5, CPU):
    PYPOSE_REFERENCE=<path to the reference checkout> python oracle/make_golden_sparse.py   # writes tests/golden/sparse.npz

Every case runs the reference's `bsr_bsc_matmul` and its `_sparse_csr_mm` dispatcher on a BSR × BSC pair (they must
agree bit for bit) and stores the inputs and the output's crow, col and values under `<case>/...`.  The shapes follow the
reference's own test (`tests/sparse/test_bsr.py`): `mT` (A is (sm, sn) blocks of (dm, dn), B is (sn, sm) blocks of
(dn, dm)) and `identical_square` (both square grids of square blocks), at zero_prob 0, 0.7 and 1.0 (that fraction of the
stored values set to zero, the blocks kept), plus empty rows and columns, a fully empty operand and an empty product.
The reference's per-pair Python loop keeps the grids at most 20 × 20 blocks.  `cases` is a JSON list of the case names.
"""
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.environ["PYPOSE_REFERENCE"])
sys.dont_write_bytecode = True
from pypose.sparse.ops import bsr_bsc_matmul, _sparse_csr_mm  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden", "sparse.npz")


def pattern(rng, rows, cols, density, empty_rows=(), empty_cols=()):
    mask = rng.random((rows, cols)) < density
    mask[list(empty_rows), :] = False
    mask[:, list(empty_cols)] = False
    return mask


def make(rng, mask, block, layout, zero_prob, dtype):
    """torch BSR (mask over block rows × block columns) or BSC (mask over block rows × block columns of the matrix)."""
    r, c = mask.shape
    if layout == "bsr":
        crow = np.concatenate([[0], np.cumsum(mask.sum(1))])
        idx = np.nonzero(mask)[1]
        ptr = crow
    else:
        ptr = np.concatenate([[0], np.cumsum(mask.sum(0))])
        idx = np.nonzero(mask.T)[1]
    val = rng.standard_normal((len(idx), *block))
    val[rng.random(val.shape) < zero_prob] = 0.0
    val = torch.from_numpy(val).to(dtype)
    ptr, idx = torch.from_numpy(ptr.astype(np.int64)), torch.from_numpy(idx.astype(np.int64))
    size = (r * block[0], c * block[1])
    f = torch.sparse_bsr_tensor if layout == "bsr" else torch.sparse_bsc_tensor
    return f(ptr, idx, val, size=size, dtype=dtype)


def main():
    rng = np.random.default_rng(20261016)
    cases, store = [], {}

    def add(name, A, B):
        C = bsr_bsc_matmul(A, B)
        C2 = _sparse_csr_mm(A, B)
        assert torch.equal(C.crow_indices(), C2.crow_indices()) and torch.equal(C.col_indices(), C2.col_indices())
        assert torch.equal(C.values(), C2.values())
        dense = A.to_dense().double() @ B.to_dense().double()
        assert torch.allclose(C.to_dense().double(), dense, atol=1e-5 if A.dtype == torch.float32 else 1e-12)
        cases.append(name)
        store.update({f"{name}/a_crow": A.crow_indices().numpy(), f"{name}/a_col": A.col_indices().numpy(),
                      f"{name}/a_val": A.values().numpy(), f"{name}/a_size": np.array(A.shape),
                      f"{name}/b_ccol": B.ccol_indices().numpy(), f"{name}/b_row": B.row_indices().numpy(),
                      f"{name}/b_val": B.values().numpy(), f"{name}/b_size": np.array(B.shape),
                      f"{name}/crow": C.crow_indices().numpy(), f"{name}/col": C.col_indices().numpy(),
                      f"{name}/val": C.values().numpy()})
        print(name, tuple(A.shape), tuple(B.shape), "nnz", A.values().shape[0], B.values().shape[0],
              C.values().shape[0], flush=True)

    for dtype, tag in ((torch.float64, "f64"), (torch.float32, "f32")):
        for zp in (0.0, 0.7, 1.0):
            for rep in range(2):
                sm, sn = (int(x) for x in rng.integers(1, 10, 2))
                dm, dn = (int(x) for x in rng.integers(1, 10, 2))
                add(f"mT_{tag}_z{zp}_{rep}",
                    make(rng, pattern(rng, sm, sn, 0.5), (dm, dn), "bsr", zp, dtype),
                    make(rng, pattern(rng, sn, sm, 0.5), (dn, dm), "bsc", zp, dtype))
                s, d = int(rng.integers(1, 10)), int(rng.integers(1, 10))
                add(f"sq_{tag}_z{zp}_{rep}",
                    make(rng, pattern(rng, s, s, 0.5), (d, d), "bsr", zp, dtype),
                    make(rng, pattern(rng, s, s, 0.5), (d, d), "bsc", zp, dtype))
        # larger grids with non-square blocks, empty rows and columns
        add(f"grid_{tag}", make(rng, pattern(rng, 20, 16, 0.3, empty_rows=(3, 7), empty_cols=(0, 5)), (3, 6), "bsr", 0.0,
                                dtype),
            make(rng, pattern(rng, 16, 18, 0.3, empty_rows=(2,), empty_cols=(4, 11)), (6, 4), "bsc", 0.0, dtype))
        add(f"blocks1_{tag}", make(rng, pattern(rng, 20, 20, 0.2), (1, 1), "bsr", 0.0, dtype),
            make(rng, pattern(rng, 20, 20, 0.2), (1, 1), "bsc", 0.0, dtype))
        add(f"blocks9_{tag}", make(rng, pattern(rng, 6, 5, 0.5), (9, 2), "bsr", 0.0, dtype),
            make(rng, pattern(rng, 5, 7, 0.5), (2, 9), "bsc", 0.0, dtype))
        # A @ A.mT
        A = make(rng, pattern(rng, 12, 15, 0.25), (4, 5), "bsr", 0.0, dtype)
        add(f"AAT_{tag}", A, A.mT)
        # a fully empty operand, and non-empty operands whose product is empty
        add(f"emptyA_{tag}", make(rng, np.zeros((5, 4), bool), (2, 3), "bsr", 0.0, dtype),
            make(rng, pattern(rng, 4, 6, 0.5), (3, 2), "bsc", 0.0, dtype))
        even = np.zeros((6, 8), bool)
        even[:, ::2] = True
        odd = np.zeros((8, 5), bool)
        odd[1::2, :] = True
        add(f"emptyC_{tag}", make(rng, even, (2, 3), "bsr", 0.0, dtype), make(rng, odd, (3, 2), "bsc", 0.0, dtype))
    store["cases"] = np.array(json.dumps(cases))
    np.savez_compressed(OUT, **store)
    print("wrote", OUT, len(cases), "cases")


if __name__ == "__main__":
    main()
