"""Every launch path of the ICP backward (csrc/knn.cu b200_icp_rec / b200_icp_bwd, module/icp.py _ICPFn) against the
fp64 model of oracle/icp_grad_oracle.py held to the matches the forward recorded, in fp32 and fp64.

The oracle replays the recorded matches instead of matching on its own, so a near-tie that fp32 resolves differently
cannot make the comparison meaningless, and the check of the returned transform pins the match store by itself.  Each
case asserts the path it reached (which paths run is decided at run time from the shapes and the SM count):

* forward: 128-thread CTAs of one query, or 256-thread CTAs of four queries when B ceil(Ns / 1024) >= 2 SMs;
* backward: nx = ceil(Ns / 1024) partial sums per batch element, folded by a 128-thread CTA (strided above 128);
* target gradient: (target row, point) pairs radix-sorted on key_bits(TB Nt) bits, TB = B for per-element targets.

Trace layout (one block per enqueued iteration): ceil(B 29 8 / 256) 256 bytes of fp64 [A_{k-1} (12) | sums (17)] per
batch element, then B Ns int32 matches, padded to 256 bytes.
"""
import ctypes
import itertools
import math

import numpy as np
import pytest
import torch

import pypose_b200 as pp
from oracle import icp_grad_oracle as O
from tests.test_pointcloud_paths_gpu import _jittered_grid, _lib_fn, _rigid, _sms, icp_nx

pytestmark = pytest.mark.gpu
DEV = "cuda"
F32, F64 = torch.float32, torch.float64
KREC = 12 + 17                         # doubles per batch element in a trace block
CHUNK_ENDS = (4, 12, 28, 60, 92)       # the device loop's host reads: chunks of 4, 8, 16, 32, 32


def fixed(K):
    """exactly K iterations of the device-decided loop"""
    return pp.utils.ReduceToBason(steps=K, patience=10 ** 6, decreasing=-math.inf, tol=-1.0)


class HostStepper(pp.utils.ReduceToBason):
    """The same rule, called by the host loop every iteration (any stepper that is not exactly ReduceToBason)."""


def host_fixed(K):
    return HostStepper(steps=K, patience=10 ** 6, decreasing=-math.inf, tol=-1.0)


# ---------------------------------------------------------------------------------------------------------------------
# paths and the recorded trace
# ---------------------------------------------------------------------------------------------------------------------
def key_bits(n):
    b = 1
    while b < 32 and (1 << b) < n:
        b += 1
    return b


def paths(B, Ns, TB, Nt):
    """-> (forward CTA shape, forward nx, backward nx, sort bits).  The forward shape is read back from the library's
    workspace size; the backward's is mirrored."""
    nx = icp_nx(B, Ns)
    small = B * -(-Ns // 1024) < 2 * _sms()
    assert nx == -(-Ns // (128 if small else 1024)), (B, Ns, nx)
    return ("small" if small else "q4"), nx, -(-Ns // 1024), key_bits(TB * Nt)


def _icp_node(T):
    seen, todo = set(), [T.tensor().grad_fn]
    while todo:
        n = todo.pop()
        if n is None or n in seen:
            continue
        if hasattr(n, "keep"):
            return n
        seen.add(n)
        todo.extend(f for f, _ in n.next_functions)
    raise AssertionError("no _ICPFn node behind the result")


def decode(T):
    """The first K recorded blocks of the forward behind T -> (A_{k-1} (K, B, 12), sums (K, B, 17), matches (K, B, Ns),
    A_K (B, 12)), all on the device."""
    ws, traces, addrs, B, Ns, Nt = _icp_node(T).keep
    K = len(addrs)
    with torch.cuda.device(0):
        blk = int(_lib_fn("b200_icp_trace_bytes", 3)(B, Ns, 1))
    ad = -(-B * KREC * 8 // 256) * 256
    assert blk == ad + -(-B * Ns * 4 // 256) * 256
    blocks = []
    for t, n in traces:
        assert t.numel() == n * blk
        blocks += [t[j * blk:(j + 1) * blk] for j in range(n)]
    assert len(blocks) >= K
    blocks = blocks[:K]
    assert [b.data_ptr() for b in blocks] == addrs          # the addresses the backward is handed
    rec = torch.stack([b[:B * KREC * 8].view(torch.float64).view(B, KREC) for b in blocks]) if K else \
        torch.zeros(0, B, KREC, dtype=torch.float64, device=DEV)
    idx = torch.stack([b[ad:ad + B * Ns * 4].view(torch.int32).view(B, Ns) for b in blocks]) if K else \
        torch.zeros(0, B, Ns, dtype=torch.int32, device=DEV)
    AK = ws[16 * 8:(16 + 12 * B) * 8].view(torch.float64).view(B, 12)
    return rec[..., :12], rec[..., 12:], idx, AK


def _rot(A):
    return A.reshape(*A.shape[:-1], 3, 4)[..., :3]


# ---------------------------------------------------------------------------------------------------------------------
# scenes: small motions, every nearest neighbour unambiguous
# ---------------------------------------------------------------------------------------------------------------------
def grid(rng, side, spacing=1.5, n=None):
    g = _jittered_grid(rng, side, spacing)
    return g[:n] if n is not None else g


def near_rows(rng, tgt, rows, angle, shift=0.05, noise=0.02):
    """Sources whose nearest targets are tgt[b, rows[b]] (tgt (1 | B, Nt, 3)), moved by one small rigid motion per
    element (tgt ~ R src + t) and clipped Gaussian noise."""
    B = rows.shape[0]
    y = np.take_along_axis(np.broadcast_to(tgt, (B,) + tgt.shape[1:]), rows[..., None], 1)
    y = y + noise * np.clip(rng.standard_normal(y.shape), -3, 3)
    R, t = _rigid(rng, B, angle, shift)
    return np.einsum("bji,bnj->bni", R, y - t[:, None])


def moved(rng, base, B, angle=0.02, shift=0.05, noise=0.01):
    """B copies of base (Ns, 3), each moved by its own small motion plus noise: (B, Ns, 3)."""
    R, t = _rigid(rng, B, angle, shift)
    return np.einsum("bij,nj->bni", R, base) + t[:, None] + noise * rng.standard_normal((B,) + base.shape)


def small_init(rng, shape, angle=0.01, shift=0.02):
    n = math.prod(shape)
    R, t = _rigid(rng, n, angle, shift)
    q = np.stack([O.mat2quat_ref(torch.from_numpy(r)).numpy() for r in R])
    return np.concatenate([t, q], 1).reshape(*shape, 7)


# ---------------------------------------------------------------------------------------------------------------------
# one run against the fixed-match oracle
# ---------------------------------------------------------------------------------------------------------------------
def icp_run(src, tgt, init, dt, st, ordv=2, req=(True, True, True)):
    s = torch.as_tensor(src).to(DEV, dt).requires_grad_(req[0])
    t = torch.as_tensor(tgt).to(DEV, dt).requires_grad_(req[1])
    i = None if init is None else pp.SE3(torch.as_tensor(init).to(DEV, dt)).requires_grad_(req[2])
    T = pp.module.ICP(stepper=st)(s, t, ord=ordv, init=i)
    return T, (s, t, i)


def cotangents(batch, seed, dt=F64):
    g = torch.Generator().manual_seed(seed)
    W = torch.randn(*batch, 4, 4, generator=g, dtype=torch.float64)
    probe = torch.randn(*batch, 5, 3, generator=g, dtype=torch.float64)
    w = torch.randn(*batch, 5, 3, generator=g, dtype=torch.float64)
    return [x.to(DEV, dt) for x in (W, probe, w)]


def kernel_loss(T, which, W, probe, w):
    return (T.matrix() * W).sum() if which == 0 else (T.unsqueeze(-2).Act(probe) * w).sum()


def rel(got, want):
    got, want = got.detach().double(), want.detach().double()
    return float((got - want).abs().max() / want.abs().max().clamp_min(1e-300))


def check(what, src, tgt, init, dt, st=None, ordv=2, seed=0):
    """Forward with grad, trace decoded, the transform and both losses' gradients against the fixed-match oracle.
    Returns (T, leaves, decoded trace, kernel gradients per loss)."""
    st = st if st is not None else pp.utils.ReduceToBason(steps=30)
    T, leaves = icp_run(src, tgt, init, dt, st, ordv)
    s, t, i = leaves
    batch = T.shape[:-1]
    B, Ns, Nt = math.prod(batch), s.shape[-2], t.shape[-2]
    A, sums, idx, AK = decode(T)
    K = st.steps
    assert A.shape[0] == K, (A.shape, K)
    assert (sums[..., 16] == Ns).all(), what                         # every source point matched once per iteration
    assert (idx >= 0).all() and (idx < Nt).all()
    Rs = [_rot(AK)] + [_rot(A[k + 1] if k + 1 < K else AK) @ _rot(A[k]).mT for k in range(K)]
    assert all(bool(O.sign_agrees(R).all()) for R in Rs), what     # both quaternion sign rules give the same graph
    matches = [idx[k].long().reshape(*batch, Ns) for k in range(K)]
    x64 = [None if x is None else (x.tensor() if isinstance(x, pp.LieTensor) else x).detach().double() for x in leaves]
    cot = cotangents(batch, seed)
    Tor, _ = O.icp(x64[0], x64[1], K, x64[2], ordv, "project", matches)
    assert float((T.tensor().detach().double() - Tor).abs().max()) <= (1e-10 if dt == F64 else 2e-5), what
    out = []
    want_leaves = [x for x in leaves if x is not None and x.requires_grad]
    for which in (0, 1):
        got = torch.autograd.grad(kernel_loss(T, which, *[c.to(dt) for c in cot]), want_leaves, retain_graph=True)
        _, ref = O.grads(x64[0], x64[1], K, x64[2], ordv, "project", *cot, which, matches)
        ref = [r for r in ref if r is not None]
        if dt == F32:
            x32 = [None if x is None else x.float() for x in x64]
            _, r32 = O.grads(x32[0], x32[1], K, x32[2], ordv, "project", *[c.float() for c in cot], which, matches)
            bounds = [max(4 * rel(a, b), 1e-6) for a, b in zip([r for r in r32 if r is not None], ref)]
        else:
            bounds = [1e-8] * len(ref)
        for name, g, r, bound in zip(("source", "target", "init"), got, ref, bounds):
            assert torch.isfinite(g).all(), (what, which, name)
            err = rel(g, r)
            print(f"\n[icp-grad] {what} {str(dt)[6:]} loss{which} {name}: K={K} err={err:.2e} bound={bound:.2e}")
            assert err <= bound, (what, which, name, err, bound)
        out.append(got)
    return T, leaves, (A, sums, idx, AK), out


DTS = [F64, F32]


# ---------------------------------------------------------------------------------------------------------------------
# the cases
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", DTS)
def test_small_ctas_ragged_backward_cta(dt):
    """B = 3, Ns = 3073 (the 4th backward CTA sums one point), Nt = 2500 (some targets matched twice)."""
    rng = np.random.default_rng(1)
    tgt = np.stack([grid(rng, 14, n=2500) for _ in range(3)])
    src = near_rows(rng, tgt, np.stack([np.arange(3073) % 2500] * 3), 0.01)
    assert paths(3, 3073, 3, 2500) == ("small", 25, 4, 13)
    check("small ragged", src, tgt, None, dt)


@pytest.mark.parametrize("dt", DTS)
def test_four_query_ctas_big_batch(dt):
    """B = 2 SMs + 16 clouds of 729 points: the recording 256 x 4 match kernel, nx = 1, more than 128 update CTAs."""
    B = 2 * _sms() + 16
    rng = np.random.default_rng(2)
    src = np.stack([grid(rng, 9) for _ in range(B)])
    tgt = np.stack([moved(rng, s, 1)[0] for s in src])
    fwd, nx, bnx, _ = paths(B, 729, B, 729)
    assert (fwd, nx, bnx) == ("q4", 1, 1) and B > 128
    check("q4 big batch", src, tgt, None, dt, ordv=math.inf)


@pytest.mark.parametrize("dt", DTS)
def test_four_query_ctas_ragged(dt):
    """B = ceil(2 SMs / 4), Ns = 4000: four 256 x 4 CTAs per element, the last one 928 points long; Nt = 3500."""
    B = -(-2 * _sms() // 4)
    rng = np.random.default_rng(3)
    tgt = np.stack([grid(rng, 16, n=3500) for _ in range(B)])
    src = near_rows(rng, tgt, np.stack([rng.permutation(4000) % 3500 for _ in range(B)]), 0.01)
    assert paths(B, 4000, B, 3500)[:3] == ("q4", 4, 4)
    check("q4 ragged", src, tgt, None, dt, ordv=1)


@pytest.mark.parametrize("dt", DTS)
def test_backward_fold_over_137_partials(dt):
    """B = 1, Ns = 140 000 against 17^3 targets: the backward's per-element fold loops over 137 partial sums."""
    rng = np.random.default_rng(4)
    tgt = grid(rng, 17, 2.0)[None]
    src = near_rows(rng, tgt, (np.arange(140000) % tgt.shape[1])[None], 0.005, noise=0.05)
    assert paths(1, 140000, 1, 4913)[2] == 137
    check("fold 137", src, tgt, None, dt, st=pp.utils.ReduceToBason(steps=12))


def _top_bit_rows(rng, Nt, n_rand):
    """Rows [0, 64) and their partners 2^16 + [0, 64) (the last rows of Nt = 2^16 + 64), interleaved as (row, partner,
    row): a sort that drops the top bit would split each row's run in two.  Plus random rows."""
    j = np.arange(64)
    return np.r_[np.stack([j, (1 << 16) + j, j], 1).reshape(-1), rng.integers(0, Nt, n_rand)]


@pytest.mark.parametrize("dt", DTS)
def test_top_sort_bit_broadcast_target(dt):
    """One target of 2^16 + 64 rows for B = 2 sources: keys use bit 16 (17-bit sort), the last 64 rows are matched,
    interleaved with the rows that share their low 16 bits."""
    rng = np.random.default_rng(5)
    Nt = (1 << 16) + 64
    tgt = grid(rng, 41, n=Nt)[None]
    rows = np.stack([_top_bit_rows(rng, Nt, 800) for _ in range(2)])
    src = near_rows(rng, tgt, rows, 0.002)
    assert paths(2, rows.shape[1], 1, Nt)[3] == 17
    _, _, (_, _, idx, _), _ = check("top bit bcast tgt", src, tgt, None, dt)
    assert int(idx.max()) == Nt - 1 and (idx >= 1 << 16).any()


@pytest.mark.parametrize("dt", DTS)
def test_top_sort_bit_per_element_target(dt):
    """Per-element targets, B = 2 x Nt = 32 800 = 2^16 + 64 keys: element 1's last rows carry bit 16.  (The sort is
    stable and element 0's points come first, so here a sort one bit short would still keep each row's run whole; the
    broadcast case above is the one whose interleaved rows tell the widths apart.)"""
    rng = np.random.default_rng(6)
    Nt = 32800
    tgt = np.stack([grid(rng, 33, n=Nt) for _ in range(2)])
    last = np.r_[np.arange(Nt - 64, Nt), np.arange(Nt - 64, Nt)]
    rows = np.stack([np.r_[last, rng.integers(0, Nt, 800)] for _ in range(2)])
    src = near_rows(rng, tgt, rows, 0.002)
    assert paths(2, rows.shape[1], 2, Nt)[3] == 17
    _, _, (_, _, idx, _), _ = check("top bit per-element tgt", src, tgt, None, dt)
    assert int(idx[:, 1].max()) == Nt - 1 and (Nt + idx[:, 1] >= 1 << 16).any()


@pytest.mark.parametrize("dt", DTS)
def test_unmatched_target_rows_get_exact_zeros(dt):
    """Ns = 100 against Nt = 200 000: the rows no iteration matched get exactly 0."""
    rng = np.random.default_rng(7)
    tgt = grid(rng, 59, n=200000)[None]
    src = near_rows(rng, tgt, rng.choice(200000, 100, replace=False)[None], 0.002)
    _, _, (_, _, idx, _), got = check("unmatched rows", src, tgt, None, dt)
    hit = torch.zeros(200000, dtype=torch.bool, device=DEV)
    hit[idx.reshape(-1).long()] = True
    assert int(hit.sum()) >= 90
    for g in got:
        assert (g[1][0][~hit] == 0).all() and (g[1][0][hit].abs().sum(-1) > 0).all()


@pytest.mark.parametrize("dt", DTS)
def test_long_scatter_runs(dt):
    """Ns = 50 000 against Nt = 64: every target row sums a run of about 780 contributions."""
    rng = np.random.default_rng(8)
    tgt = grid(rng, 4)[None]
    src = near_rows(rng, tgt, (rng.permutation(50000) % 64)[None], 0.02, noise=0.05)
    check("long runs", src, tgt, None, dt)


BCASTS = ["source", "target", "init1", "initB"]


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("shape", ["small", "q4"])
@pytest.mark.parametrize("kind", BCASTS)
def test_broadcast_sums(kind, shape, dt):
    """Stride-0 source, target or (1, 7) init summed over the batch, and a per-element (B, 7) init, on both CTA shapes."""
    B = 3 if shape == "small" else 2 * _sms() + 16
    rng = np.random.default_rng(10 + BCASTS.index(kind))
    base = grid(rng, 9)
    one, many = base[None], moved(rng, base, B)
    src, tgt, init = {"source": (one, many, None), "target": (many, one, None)}.get(kind, (None, None, None))
    if kind.startswith("init"):
        src = np.stack([grid(rng, 9) for _ in range(B)])
        tgt = np.stack([moved(rng, s, 1)[0] for s in src])
        init = small_init(rng, (1,) if kind == "init1" else (B,))
    assert paths(B, 729, B, 729)[0] == shape
    check(f"bcast {kind} {shape}", src, tgt, init, dt, st=pp.utils.ReduceToBason(steps=20), seed=1)


@pytest.mark.parametrize("dt", DTS)
def test_two_dimensional_broadcast_batch(dt):
    """Source (2, 1), target (1, 3) and init (3, 7): all three are expanded to the six elements of the (2, 3) batch
    before the kernels run, and autograd sums the gradients back over the expands."""
    rng = np.random.default_rng(20)
    base = grid(rng, 8)
    src = (base[None] + 0.01 * rng.standard_normal((2,) + base.shape))[:, None]
    tgt = moved(rng, base, 3, noise=0.0)[None]
    init = small_init(rng, (3,))
    T, *_ = check("batch (2,1)x(1,3)", src, tgt, init, dt)
    assert T.shape == (2, 3, 7)


# ---------------------------------------------------------------------------------------------------------------------
# which operands want a gradient, and the cotangent
# ---------------------------------------------------------------------------------------------------------------------
def _subset_scene():
    rng = np.random.default_rng(30)
    src = np.stack([grid(rng, 9) for _ in range(3)])
    tgt = np.stack([moved(rng, s, 1)[0] for s in src])
    return src, tgt, small_init(rng, (3,))


@pytest.mark.parametrize("dt", DTS)
def test_every_requires_grad_subset_is_bit_identical(dt):
    src, tgt, init = _subset_scene()
    W, probe, w = cotangents((3,), 31, dt)
    full = None
    for req in [(True, True, True)] + [r for r in itertools.product((True, False), repeat=3) if any(r) and not all(r)]:
        T, leaves = icp_run(src, tgt, init, dt, fixed(9), req=req)
        got = iter(torch.autograd.grad(kernel_loss(T, 1, W, probe, w), [x for x, r in zip(leaves, req) if r]))
        g = [next(got) if r else None for r in req]
        if full is None:
            full = g
        for a, b in zip(g, full):
            assert a is None or torch.equal(a, b), req


@pytest.mark.parametrize("dt", DTS)
def test_zero_and_translation_only_cotangents(dt):
    src, tgt, init = _subset_scene()
    T, leaves = icp_run(src, tgt, init, dt, fixed(9))
    for g in torch.autograd.grad((T.tensor() * 0).sum(), leaves, retain_graph=True):
        assert (g == 0).all()
    v = cotangents((3,), 32)[1][:, 0].contiguous()
    got = torch.autograd.grad((T.tensor()[..., :3] * v.to(dt)).sum(), leaves)
    _, _, idx, _ = decode(T)
    x64 = [torch.as_tensor(x).to(DEV, dt).double().requires_grad_() for x in (src, tgt, init)]
    Tor, _ = O.icp(x64[0], x64[1], 9, x64[2], matches=[m.long() for m in idx])
    ref = torch.autograd.grad((Tor[..., :3] * v).sum(), x64)
    for a, b in zip(got, ref):
        assert rel(a, b) <= (1e-8 if dt == F64 else 1e-5), rel(a, b)


# ---------------------------------------------------------------------------------------------------------------------
# iteration plumbing: chunk edges, a tolerance stop inside a chunk, K = 0
# ---------------------------------------------------------------------------------------------------------------------
def _plumbing_scene(slow=False):
    rng = np.random.default_rng(40)
    src = np.stack([grid(rng, 9) for _ in range(3)])
    tgt = np.stack([moved(rng, s, 1)[0] for s in src])
    if slow:                              # element 0: a larger turn, converging over more steps
        R, _ = _rigid(rng, 1, 0.15, 0.0)
        tgt[0] = src[0] @ R[0].T + np.array([0.3, -0.2, 0.1]) + 0.01 * rng.standard_normal(src[0].shape)
    return src, tgt


def _device_equals_host(src, tgt, dt, dev_st, host_st):
    a, la = icp_run(src, tgt, None, dt, dev_st)
    b, lb = icp_run(src, tgt, None, dt, host_st)
    assert dev_st.steps == host_st.steps
    assert torch.equal(a.tensor(), b.tensor())
    W, probe, w = cotangents((3,), 41, dt)
    for which in (0, 1):
        ga = torch.autograd.grad(kernel_loss(a, which, W, probe, w), la[:2], retain_graph=True)
        gb = torch.autograd.grad(kernel_loss(b, which, W, probe, w), lb[:2], retain_graph=True)
        assert all(torch.equal(x, y) for x, y in zip(ga, gb)), which
    return dev_st.steps


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("K", [1, 3, 4, 5, 12, 13, 28, 29, 60, 61])
def test_fixed_iterations_device_loop_equals_host_loop(K, dt):
    """Trace blocks addressed per chunk (device loop) and one per call (host loop) give the same gradients bit for bit;
    the first iteration of each new chunk also against the oracle."""
    src, tgt = _plumbing_scene()
    assert _device_equals_host(src, tgt, dt, fixed(K), host_fixed(K)) == K
    if K in (1, 5, 13, 29, 61):
        check(f"K={K}", src, tgt, None, dt, st=fixed(K))


@pytest.mark.parametrize("dt", DTS)
def test_tolerance_stop_inside_a_chunk(dt):
    """A stop on tol after a step that ends no chunk: the rest of the chunk's blocks stay unwritten and unread."""
    src, tgt = _plumbing_scene(slow=True)
    losses = []

    class Rec(HostStepper):
        def step(self, loss):
            losses.append(float(loss.max()))
            super().step(loss)

    icp_run(src, tgt, None, dt, Rec(steps=20, patience=10 ** 6, decreasing=-math.inf, tol=-1.0))
    cands = [s for s in range(2, 12) if s not in CHUNK_ENDS and losses[s - 1] < min(losses[:s - 1])]
    assert cands, losses
    s = cands[-1]
    tol = (losses[s - 1] + min(losses[:s - 1])) / 2
    mk = lambda cls: cls(steps=61, patience=10 ** 6, decreasing=-math.inf, tol=tol)   # noqa: E731
    assert _device_equals_host(src, tgt, dt, mk(pp.utils.ReduceToBason), mk(HostStepper)) == s
    st = mk(pp.utils.ReduceToBason)
    check(f"tol stop at {s}", src, tgt, None, dt, st=st)
    assert st.steps == s


def _ptr(t):
    return None if t is None else t.data_ptr()


@pytest.mark.parametrize("dt", DTS)
def test_zero_iterations_through_the_c_abi(dt):
    """b200_icp_rec with 0 iterations leaves A = init; b200_icp_bwd with K = 0 differentiates svdtf(source, init
    source) only, and the target gets exact zeros."""
    from pypose_b200 import _C
    rng = np.random.default_rng(50)
    B, Ns, Nt = 2, 700, 729
    src = torch.from_numpy(np.stack([grid(rng, 9)[:Ns] for _ in range(B)])).to(DEV, dt).contiguous()
    tgt = torch.from_numpy(np.stack([grid(rng, 9) for _ in range(B)])).to(DEV, dt).contiguous()
    init = torch.from_numpy(small_init(rng, (B,), 0.3, 0.5)).to(DEV, dt).contiguous()
    sfx = _C.suffix(dt)
    with torch.cuda.device(0):
        ws = torch.empty(int(_lib_fn("b200_icp_workspace_bytes", 2)(B, Ns)), dtype=torch.uint8, device=DEV)
        out, err, last = (torch.empty(B, 7, dtype=dt, device=DEV), torch.empty(B, dtype=dt, device=DEV),
                          torch.empty(B, dtype=dt, device=DEV))
        _C.check(_C.fn(f"b200_icp_rec_{sfx}")(src.data_ptr(), Ns * 3, tgt.data_ptr(), Nt * 3, init.data_ptr(), 7,
                                               out.data_ptr(), err.data_ptr(), last.data_ptr(), ws.data_ptr(), B, Ns, Nt,
                                               2, 1, 0, 0, 0, 0, 0.0, 0.0, None, 0, None, _C.stream_ptr(src.device)),
                 "rec")
        x64 = [x.double().requires_grad_() for x in (src, tgt, init)]
        Tor, m = O.icp(x64[0], x64[1], 0, x64[2])
        assert m == [] and float((out.double() - Tor).abs().max()) <= (1e-10 if dt == F64 else 2e-6)
        bws = torch.empty(int(_lib_fn("b200_icp_bwd_workspace_bytes", 4)(B, Ns, Nt, B)), dtype=torch.uint8, device=DEV)
        for which in (0, 1):
            cot = cotangents((B,), 51 + which)
            o = out.double().requires_grad_()
            gout, = torch.autograd.grad(O.losses(o, *cot)[which], [o])
            gout = gout.to(dt).contiguous()
            gs, gt, gi = torch.empty_like(src), torch.full_like(tgt, float("nan")), torch.empty_like(init)
            arr = (ctypes.c_longlong * 1)()
            _C.check(_C.fn(f"b200_icp_bwd_{sfx}")(src.data_ptr(), Ns * 3, tgt.data_ptr(), Nt * 3, init.data_ptr(), 7,
                                                   ws.data_ptr(), arr, 0, gout.data_ptr(), gs.data_ptr(), gt.data_ptr(),
                                                   gi.data_ptr(), bws.data_ptr(), B, Ns, Nt, _C.stream_ptr(src.device)),
                     "bwd")
            rs, ri = torch.autograd.grad(O.losses(O.icp(x64[0], x64[1], 0, x64[2])[0], *cot)[which], [x64[0], x64[2]])
            assert (gt == 0).all()
            tol = 1e-8 if dt == F64 else 1e-5
            assert rel(gi, ri) <= tol, (which, rel(gi, ri))
            # T = svdtf(s, init s) is init whatever s is: the source gradient is rounding, held to the init's scale
            assert float((gs.double() - rs).abs().max()) <= tol * float(ri.abs().max()), which


# ---------------------------------------------------------------------------------------------------------------------
# isolation and reproducibility
# ---------------------------------------------------------------------------------------------------------------------
def test_big_batch_elements_get_the_gradients_they_get_alone():
    """fp64, 8 iterations: elements {0, 1, B/2, B - 1} of the 256 x 4 batch (Ns = 700 != Nt = 729) and the same element
    alone (B = 1, 128-thread CTAs) agree to 1e-12: same matches, no leak between elements' target rows."""
    B = 2 * _sms() + 16
    rng = np.random.default_rng(60)
    tgt = np.stack([grid(rng, 9) for _ in range(B)])
    src = near_rows(rng, tgt, np.stack([rng.permutation(729)[:700] for _ in range(B)]), 0.01)
    assert paths(B, 700, B, 729)[0] == "q4" and paths(1, 700, 1, 729)[0] == "small"
    W, probe, w = cotangents((B,), 61)
    T, (s, t, _) = icp_run(src, tgt, None, F64, fixed(8))
    gb = torch.autograd.grad(kernel_loss(T, 0, W, probe, w) + kernel_loss(T, 1, W, probe, w), [s, t])
    for b in (0, 1, B // 2, B - 1):
        T1, (s1, t1, _) = icp_run(src[b:b + 1], tgt[b:b + 1], None, F64, fixed(8))
        c = [x[b:b + 1] for x in (W, probe, w)]
        g1 = torch.autograd.grad(kernel_loss(T1, 0, *c) + kernel_loss(T1, 1, *c), [s1, t1])
        for x, y in zip(gb, g1):
            assert rel(x[b:b + 1], y) <= 1e-12, (b, rel(x[b:b + 1], y))


@pytest.mark.parametrize("dt", DTS)
def test_four_query_backward_is_bit_reproducible(dt):
    B = 2 * _sms() + 16
    rng = np.random.default_rng(70)
    src = np.stack([grid(rng, 9) for _ in range(B)])
    tgt = np.stack([moved(rng, s, 1)[0] for s in src])
    assert paths(B, 729, B, 729)[0] == "q4"
    T, leaves = icp_run(src, tgt, None, dt, fixed(10))
    W, probe, w = cotangents((B,), 71, dt)
    L = kernel_loss(T, 0, W, probe, w)
    a = torch.autograd.grad(L, leaves[:2], retain_graph=True)
    b = torch.autograd.grad(L, leaves[:2])
    assert all(torch.isfinite(x).all() and torch.equal(x, y) for x, y in zip(a, b))
