"""Parity of the size-selected kernel routes against high-precision references, on both sides of every threshold.

The library picks kernels by size: `mmssl_spmm_csr_f32` with impl 0 switches to the register-capped kernel (6 blocks per SM, epilogue
table loads after the gathers) at 2^21 COO entries and drops the evict-last policy of the gathered table above 96 MiB; InfoNCE runs on
the tensor cores for n <= 2048 and d in {64, 128} and on the CUDA cores otherwise.  The big configurations take the large side of
each threshold, so each side is compared here with a float64 reference: scipy for SpMM, autograd of `oracle.mmssl_oracle.infonce`
for InfoNCE.  The bodies are `check_*` functions that take their sizes; tests/test_emu_route_parity.py runs them at small sizes on
the CPU emulator."""
import math

import numpy as np
import pytest
import scipy.sparse as sp
import torch
import torch.nn.functional as F
from torch.utils.checkpoint import checkpoint

from tests.golden_util import rel_err

pytestmark = pytest.mark.gpu

SPMM_AUTO_NNZ = 1 << 21                 # impl 0: register-capped kernel from this many COO entries (duplicates count)
X_POLICY_FLOATS = (96 << 20) // 4       # gathered tables above this many floats are not marked evict-last
HEAVY_ROW = 1024                        # plan: rows over this many non-zeros are reduced with vector atomics


def _note(worst, key, err):
    """Keeps the largest error of `key` in the check's own dict; _report prints them (pytest -s)."""
    worst[key] = max(worst.get(key, 0.0), float(err))
    return err


def _report(worst):
    for k in sorted(worst):
        print(f"{k}: {worst[k]:.3g}")


def _cached(graphs, key, build):
    """`graphs`: a dict owned by the caller (a module-scoped fixture on the GPU), or None to build afresh.  A graph holds device
    pointers and work areas of the device it was built on, so the emulated tests never share one."""
    if graphs is None:
        return build()
    if key not in graphs:
        graphs[key] = build()
    return graphs[key]


def _mm(ref, x):
    """float64 scipy product ref @ x"""
    return torch.from_numpy(ref @ x.detach().double().cpu().numpy())


def _graph_from_coo(r, c, v, shape):
    from mmssl_b200.graph import BipartiteGraph
    ref = sp.coo_matrix((v.astype(np.float64), (r, c)), shape=shape).tocsr()      # duplicates summed
    g = BipartiteGraph(torch.from_numpy(r).cuda(), torch.from_numpy(c).cuda(), torch.from_numpy(v).cuda(), shape)
    return g, ref


def _zipf(rng, n, size, s):
    p = 1.0 / np.arange(1, n + 1) ** s
    return rng.permutation(n)[rng.choice(n, size, p=p / p.sum())]


def zipf_graph(nnz, n_rows, n_cols, seed=0):
    """`nnz` COO entries (duplicates included): uniform rows, Zipf columns -- A^T has a few very long rows, as the item rows
    of a power-law graph do.  Values are random signs scaled by 1 / sqrt(column degree), like the normalised graph, so the
    50k-term rows stay of order one and the softmax epilogue sees logits of the size it sees in training."""
    rng = np.random.default_rng(seed)
    r = rng.integers(0, n_rows, nnz)
    c = _zipf(rng, n_cols, nnz, 1.0)
    v = (rng.standard_normal(nnz) / np.sqrt(np.bincount(c, minlength=n_cols)[c])).astype(np.float32)
    return _graph_from_coo(r, c, v, (n_rows, n_cols))


def cut_graph(seed=0):
    """300 x 200, about 6.5k COO entries, laid out on the cuts of the default plan: rows of exactly 1025 (heavy), 64 (whole),
    1024 (longest split row that is not heavy) and 65 (shortest split row) non-zeros, a 1500-entry heavy row, seven empty rows,
    short random rows; Zipf columns give A^T rows over 1024 as well.  The long rows come first, so the split rows start
    at non-zero offsets."""
    rng = np.random.default_rng(seed)
    n_rows, n_cols = 300, 200
    lens = np.zeros(n_rows, np.int64)
    lens[:5] = [1025, 64, 1024, 65, 1500]
    lens[12:] = rng.integers(0, 21, n_rows - 12)       # rows 5..11 stay empty
    r = np.repeat(np.arange(n_rows), lens)
    c = _zipf(rng, n_cols, len(r), 1.2)
    v = rng.standard_normal(len(r)).astype(np.float32)
    perm = rng.permutation(len(r))
    return _graph_from_coo(r[perm], c[perm], v[perm], (n_rows, n_cols))


def _row_lengths(a):
    return (a.rowptr[1:] - a.rowptr[:-1]).cpu()


def _work_area_clean(a, width):
    """The arrival counters and the heavy rows' accumulation slots are left zero after every launch."""
    part, cnt = a.work_area(width)
    assert int(cnt.count_nonzero()) == 0
    st = a.split_table[:4 * a.n_split_rows].view(-1, 4).cpu()
    slots = st[st[:, 3] != 0, 0].long()
    if len(slots):
        assert float(part.view(-1, width)[slots.cuda()].abs().max()) == 0.0


def _check_operand(a, ref, d, nrhs, impl, gen, key, tol, tol_sm, worst, peers=False, repeat_light=False):
    """Every epilogue of one operand, twice, against float64: plain, +alpha*C then softmax with a running-sum base (s_mode 2),
    accumulate into the running sum (s_mode 1), softmax backward, C aliasing Y; optionally the peer-table stores (y_mode 2) and
    bitwise repeatability of the rows the plan reduces in a fixed order."""
    from mmssl_b200 import ops
    m, k = ref.shape
    wide = torch.randn(k, nrhs * d + 8, generator=gen).cuda()
    xs = [wide[:, r * d:(r + 1) * d] for r in range(nrhs)]         # strided views (ld != d)
    cs = [torch.randn(m, d, generator=gen).cuda() for _ in range(nrhs)]
    sb = [torch.randn(m, d, generator=gen).cuda() for _ in range(nrhs)]
    ysv = [torch.softmax(torch.randn(m, d, generator=gen), -1).cuda() for _ in range(nrhs)]
    base = [_mm(ref, x) for x in xs]
    cd, sbd = [c.double().cpu() for c in cs], [t.double().cpu() for t in sb]
    sm = [torch.softmax(b + 0.25 * c, -1) for b, c in zip(base, cd)]
    want_s2 = [t + w for t, w in zip(sbd, sm)]
    want_s1 = [t + b + 0.5 * c for t, b, c in zip(want_s2, base, cd)]
    want_bwd = []
    for yv, b, c in zip(ysv, base, cd):
        v, yd = b + 0.25 * c, yv.double().cpu()
        want_bwd.append(yd * (v - (v * yd).sum(-1, keepdim=True)))
    want_acc = [b + c for b, c in zip(base, cd)]
    for _ in range(2):
        for y, want in zip(ops.spmm(a, xs, impl=impl), base):
            assert _note(worst, key + " plain", rel_err(y, want)) < tol
        _work_area_clean(a, nrhs * d)
        s = [torch.empty(m, d).cuda() for _ in range(nrhs)]
        ys = ops.spmm(a, xs, cs=cs, alpha=0.25, epilogue=ops.EPI_SOFTMAX, ss=s, s_mode=2, sbases=sb, impl=impl)
        for y, si, want, w2 in zip(ys, s, sm, want_s2):
            assert _note(worst, key + " softmax", rel_err(y, want)) < tol_sm
            assert _note(worst, key + " softmax", rel_err(si, w2)) < tol_sm
        ops.spmm(a, xs, cs=cs, alpha=0.5, epilogue=ops.EPI_NONE, ss=s, s_mode=1, impl=impl)
        for si, w1 in zip(s, want_s1):
            assert _note(worst, key + " s_mode 1", rel_err(si, w1)) < tol_sm
        ts = ops.spmm(a, xs, cs=cs, alpha=0.25, epilogue=ops.EPI_SOFTMAX_BWD, ysaved=ysv, impl=impl)
        for t, want in zip(ts, want_bwd):
            assert _note(worst, key + " softmax bwd", rel_err(t, want)) < tol
        acc = [c.clone() for c in cs]
        ops.spmm(a, xs, acc, cs=acc, alpha=1.0, impl=impl)         # C aliases Y
        for y, want in zip(acc, want_acc):
            assert _note(worst, key + " C aliases Y", rel_err(y, want)) < tol
        _work_area_clean(a, nrhs * d)
    if peers:       # y_mode 2 with two local buffers standing in for the peer-mapped tables
        ys = [torch.empty(m, d).cuda() for _ in range(nrhs)]
        pt = [[torch.full((m, d), float("nan")).cuda() for _ in range(2)] for _ in range(nrhs)]
        ops.spmm(a, xs, ys, impl=impl, y_mode=2, y_peers=[[t.data_ptr() for t in q] for q in pt])
        for y, q, b in zip(ys, pt, base):
            assert rel_err(y, b) < tol
            for t in q:
                assert torch.equal(t, y)
    if repeat_light:        # rows up to 1024 non-zeros are reduced in a fixed order: bitwise repeatable
        light = (_row_lengths(a) <= HEAVY_ROW).cuda()
        y1, y2 = ops.spmm(a, xs, impl=impl), ops.spmm(a, xs, impl=impl)
        for u, w in zip(y1, y2):
            assert torch.equal(u[light], w[light])


def check_spmm_auto_route(nnz, n_rows, n_cols, d, nrhs, impl=0, min_heavy=50_000, seed=0, graphs=None):
    """A Zipf graph of `nnz` COO entries, both operands, every epilogue, with impl 0 (the automatic route) or an explicit impl."""
    g, ref = _cached(graphs, ("zipf", nnz, n_rows, n_cols, seed), lambda: zipf_graph(nnz, n_rows, n_cols, seed))
    # impl 0 compares the nnz of the descriptor the kernel receives with 2^21: it must be the COO count, duplicates included
    for a in (g.fwd, g.bwd):
        assert int(a.desc.nnz) == nnz and int(a.rowptr[-1]) == nnz
    assert int(_row_lengths(g.bwd).max()) >= min_heavy
    gen = torch.Generator().manual_seed(seed + d + nrhs)
    worst = {}
    # the A^T rows of 50k+ non-zeros are summed with float atomics in arrival order, so their error changes from run to run
    for a, r, side in ((g.fwd, ref, "A"), (g.bwd, ref.T.tocsr(), "A^T")):
        _check_operand(a, r, d, nrhs, impl, gen, f"spmm impl {impl} nnz={nnz} d={d} nrhs={nrhs} {side}", 1e-5, 1e-4, worst)
    _report(worst)


def check_spmm_variant(impl, d, nrhs, seed=0, graphs=None):
    """One LDG-kernel variant on the plan-cut graph against float64, both operands, peer stores, bitwise repeatability."""
    g, ref = _cached(graphs, ("cut", seed), lambda: cut_graph(seed))
    lens = _row_lengths(g.fwd)
    assert sorted(lens[:5].tolist()) == [64, 65, 1024, 1025, 1500] and int((lens == 0).sum()) >= 7
    assert int(_row_lengths(g.bwd).max()) > HEAVY_ROW
    gen = torch.Generator().manual_seed(seed + impl + d + nrhs)
    worst = {}
    for a, r, side in ((g.fwd, ref, "A"), (g.bwd, ref.T.tocsr(), "A^T")):
        _check_operand(a, r, d, nrhs, impl, gen, f"spmm impl {impl} d={d} nrhs={nrhs} {side}", 3e-6, 3e-5, worst,
                       peers=True, repeat_light=True)
    _report(worst)


# ------------------------------------------------------------------------------------------------------------ InfoNCE
def _infonce_ref_blockwise(a, b, tau, block):
    """oracle.infonce's formula on normalised rows, one row block at a time under activation checkpointing: the backward
    recomputes a block's similarity rows instead of keeping all n x n of them."""
    def rows(a, b, lo):
        hi = min(lo + block, a.shape[0])
        refl = torch.exp(a[lo:hi] @ a.t() / tau)
        betw = torch.exp(a[lo:hi] @ b.t() / tau)
        dr, db = refl[:, lo:hi].diagonal(), betw[:, lo:hi].diagonal()
        return (-torch.log(db / (refl.sum(1) + betw.sum(1) - dr) + 1e-8)).sum()
    tot = 0.0
    for lo in range(0, a.shape[0], block):
        tot = tot + checkpoint(rows, a, b, lo, use_reentrant=False)
    return tot / a.shape[0]


def infonce_reference(t1, t2, idx, tau, g_loss, block=None):
    """float64 autograd of  g_loss * infonce(t1[idx], t2[idx]) on the device of t1: (loss, d/dt1, d/dt2)"""
    from oracle import mmssl_oracle as O
    T1, T2 = t1.double().requires_grad_(True), t2.double().requires_grad_(True)
    if block is None:
        loss = O.infonce(T1[idx], T2[idx], O.HotPathConfig(embed_size=t1.shape[1], tau=tau))
    else:
        loss = _infonce_ref_blockwise(F.normalize(T1[idx]), F.normalize(T2[idx]), tau, block)
    (g_loss * loss).backward()
    return float(loss.detach()), T1.grad, T2.grad


def check_infonce(n, d, tau, impl, seed=0, ref_block=None):
    """One InfoNCE evaluation as the hot step issues it: rows gathered through `idx` with duplicates from strided views of
    [U, 2d + 4] tables (one table row zero), a device g_loss != 1, gradients added into pre-filled strided gradient tables.
    Work buffers start as NaN, so a kernel that reads what it did not write shows."""
    from mmssl_b200 import ops
    gen = torch.Generator().manual_seed(1000 * seed + n + d)
    U = max(n // 2, 1) + 3                                        # fewer table rows than batch rows: users repeat
    idx = torch.randint(0, U, (n,), generator=gen)
    if n >= 2:
        idx[n - 1] = idx[0]
    # a zero table row in the batch (normalize's eps path); at n = 1 outside it: the one row's exact gradient is 0, and g / eps
    # would turn the fp32 residue of that 0 into 1e6
    zero_user = int(idx[n // 2]) if n >= 2 else (int(idx[0]) + 1) % U
    w1, w2 = torch.randn(U, 2 * d + 4, generator=gen), 0.5 * torch.randn(U, 2 * d + 4, generator=gen)
    w1[zero_user, :d] = 0
    idx_d, g_loss = idx.cuda(), torch.tensor([1.7]).cuda()
    dev = idx_d.device
    want, r1, r2 = infonce_reference(w1[:, :d].to(dev), w2[:, d + 4:].to(dev), idx_d, tau, 1.7, ref_block)
    r1, r2 = r1.cpu(), r2.cpu()
    others = torch.ones(U, dtype=torch.bool)
    others[zero_user] = False
    # gradient tables pre-filled with values of the size of the gradient (larger ones would round away what is added); the
    # zero row's gradient is g / eps, 1e12 times the others, so it gets its own scale and is compared on its own
    s1, s2 = float(r1[others].abs().max()) + 1e-30, float(r2.abs().max()) + 1e-30
    g1, g2 = s1 * torch.randn(U, 2 * d + 4, generator=gen), s2 * torch.randn(U, 2 * d + 4, generator=gen)
    g1[zero_user] = (float(r1[zero_user].abs().max()) + 1e-30) * torch.randn(2 * d + 4, generator=gen)
    W1, W2, G1, G2 = w1.cuda(), w2.cuda(), g1.cuda(), g2.cuda()
    z1, z2 = W1[:, :d], W2[:, d + 4:]
    gz1, gz2 = G1[:, d + 4:], G2[:, :d]
    work = ops.InfoNCEWork(n, d, idx_d.device, impl=impl)
    assert work.tc == (impl == "auto" and n <= 2048 and d in (64, 128))
    for t in (work.a, work.b, work.na, work.nb, work.ga, work.gb, work.stats, work.coef, work.loss_part):
        t.fill_(float("nan"))
    if work.ws is not None:
        work.ws.fill_(0xFF)
    part = ops.infonce_forward(z1, z2, idx_d, 1.0 / tau, work, g_loss=g_loss)
    ops.infonce_backward(idx_d, 1.0 / tau, work, gz1, gz2)
    got = float(part.double().sum()) / n
    key = f"infonce {'tc' if work.tc else 'simt'} d={d} n={n} tau={tau}"
    # n = 1: the exact loss is -1e-8 and the exact gradients are 0 (the one ratio is B / (R + B - R) = 1), but R_ii = e^(1 / tau)
    # cancels in fp32 and leaves a few ulps of it -- measured 2.3e-5 in the loss and 4e-6 in the gradients at tau = 0.5.  The
    # tensor-core backward keeps R_ii only to its bf16 hi / lo precision (2^-17), which leaves 2^-17 e^(1 / tau) g_loss / (tau |z|)
    # in the gradient: 1.2e-3 at tau = 0.2, d = 64 (measured 1.1e-3).  The floor, 2^-16 e^(1 / tau), is above both; it is zero for
    # n > 1.
    floor = 2.0 ** -16 * math.exp(1.0 / tau) if n == 1 else 0.0
    worst = {}
    if n == 1:      # against the floor: a relative error to -1e-8 says nothing
        assert _note(worst, key + " loss, absolute", abs(got - want)) < floor, (got, want)
    else:
        assert _note(worst, key + " loss", abs(got - want) / abs(want)) < 1e-4, (got, want)
    G1c, G2c = G1.cpu(), G2.cpu()
    # the other columns of the strided gradient tables are not touched
    assert torch.equal(G1c[:, :d + 4], g1[:, :d + 4]) and torch.equal(G2c[:, d:], g2[:, d:])
    d1, d2 = (G1c[:, d + 4:].double() - g1[:, d + 4:].double()), (G2c[:, :d].double() - g2[:, :d].double())
    for got_g, want_g, name in ((d1[others], r1[others], "dz1"), (d1[zero_user], r1[zero_user], "dz1 zero row"), (d2, r2, "dz2")):
        err = float((got_g - want_g).abs().max())
        scale = float(want_g.abs().max())
        if n == 1:
            _note(worst, key + " " + name + ", absolute", err)
        else:
            _note(worst, key + " " + name, err / (scale + 1e-30))
        assert err <= 1e-4 * scale + floor, (name, err, scale)
    _report(worst)
    return work


def check_nce_streams_bitwise(n, d, tau=0.5, seed=0):
    """Tensor-core backward: the three products on two side streams (ops.NCE_STREAMS) give the bits of phase -1 on one stream."""
    from mmssl_b200 import ops
    gen = torch.Generator().manual_seed(seed + n)
    z1, z2 = torch.randn(n, d, generator=gen).cuda(), torch.randn(n, d, generator=gen).cuda()
    work = ops.InfoNCEWork(n, d, z1.device, impl="auto")
    assert work.tc
    ops.infonce_forward(z1, z2, None, 1.0 / tau, work)
    out = []
    old = ops.NCE_STREAMS
    try:
        for streams in (True, False):
            ops.NCE_STREAMS = streams
            work.ga.fill_(float("nan")); work.gb.fill_(float("nan"))
            ops.infonce_backward(None, 1.0 / tau, work, None, None)
            torch.cuda.synchronize()
            out.append((work.ga.clone(), work.gb.clone()))
    finally:
        ops.NCE_STREAMS = old
    assert torch.equal(out[0][0], out[1][0]) and torch.equal(out[0][1], out[1][1])


# --------------------------------------------------------------------------------------------------------------- tests
_BIG = 140_000      # rows and columns of the 2^21-entry graphs: n * d * nrhs > 96 MiB of gathered table on both operands


@pytest.fixture(scope="module")
def graphs():
    """The graphs of this module's tests, built once on the device (the 2^21-entry ones take seconds to build and to
    reference); dropped with the module."""
    cache = {}
    yield cache
    cache.clear()


@pytest.mark.parametrize("nnz", [SPMM_AUTO_NNZ - 1, SPMM_AUTO_NNZ])
@pytest.mark.parametrize("d,nrhs", [(64, 3), (128, 2), (256, 1)])
def test_spmm_auto_route_threshold(graphs, nnz, d, nrhs):
    """impl 0 on both sides of 2^21 entries (the 128-thread kernel below, the register-capped one from there on)."""
    check_spmm_auto_route(nnz, _BIG, _BIG, d, nrhs, graphs=graphs)


@pytest.mark.parametrize("impl,d,nrhs", [(128, 128, 2), (256, 64, 3), (256, 256, 1)])
def test_spmm_hint_variants_large(graphs, impl, d, nrhs):
    """The L2-hint variants where their policy matters: 2^21 entries and a gathered table above 96 MiB, so the gathers are
    issued with the "no preference" policy instead of evict-last (impl 0 does not read the policy)."""
    assert _BIG * d * nrhs > X_POLICY_FLOATS
    check_spmm_auto_route(SPMM_AUTO_NNZ, _BIG, _BIG, d, nrhs, impl=impl, graphs=graphs)


VARIANTS = [8, 16, 24, 2 | 8, 2 | 16, 16 | 64, 128, 256]


@pytest.mark.parametrize("impl", VARIANTS)
@pytest.mark.parametrize("d,nrhs", [(64, 1), (64, 3), (128, 2), (256, 1), (256, 3)])
def test_spmm_variant_vs_fp64(graphs, impl, d, nrhs):
    check_spmm_variant(impl, d, nrhs, graphs=graphs)


NCE_N = [1, 2, 63, 64, 65, 127, 128, 129, 1023, 1025, 2047, 2048]


@pytest.mark.parametrize("impl", ["auto", "simt"])
@pytest.mark.parametrize("n", NCE_N)
@pytest.mark.parametrize("d", [64, 128])
@pytest.mark.parametrize("tau", [0.2, 0.5, 1.0])
def test_infonce_routes(impl, n, d, tau):
    check_infonce(n, d, tau, impl)


@pytest.mark.parametrize("n,d", [(96, 256), (1024, 256), (2049, 256), (2049, 64), (4096, 64), (4096, 128), (16384, 64), (16384, 128)])
@pytest.mark.parametrize("tau", [0.2, 0.5, 1.0])
def test_infonce_cuda_core_route(n, d, tau):
    """Above 2048 rows, and at d = 256, the automatic route is the CUDA-core one."""
    work = check_infonce(n, d, tau, "auto", ref_block=1024 if n > 4096 else None)
    assert not work.tc


@pytest.mark.parametrize("n,d", [(128, 64), (1025, 64), (2048, 128)])
def test_infonce_tc_streams_bitwise(n, d):
    check_nce_streams_bitwise(n, d)
