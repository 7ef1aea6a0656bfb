"""Per-kernel parity of libmmssl_b200 against CPU restatements (scipy / torch-CPU fp64).  All tests
call through the C ABI (ctypes) on a real H100."""
import math

import numpy as np
import pytest
import scipy.sparse as sp
import torch

pytestmark = pytest.mark.gpu

from tests.golden_util import rel_err  # noqa: E402


def _dev():
    return torch.device("cuda")


def _rand_graph(n_rows, n_cols, nnz, seed, heavy_rows=0, dup=True):
    rng = np.random.default_rng(seed)
    r = rng.integers(0, n_rows, nnz)
    c = rng.integers(0, n_cols, nnz)
    if heavy_rows:   # a few very long rows -> split segments
        k = nnz // 3
        r[:k] = rng.integers(0, heavy_rows, k)
    if not dup:
        key = np.unique(r.astype(np.int64) * n_cols + c)
        r, c = key // n_cols, key % n_cols
    v = rng.standard_normal(len(r)).astype(np.float32)
    perm = rng.permutation(len(r))
    return r[perm].astype(np.int64), c[perm].astype(np.int64), v[perm]


def _graph(n_rows, n_cols, nnz, seed, heavy_rows=0):
    from mmssl_b200.graph import BipartiteGraph
    r, c, v = _rand_graph(n_rows, n_cols, nnz, seed, heavy_rows)
    ref = sp.coo_matrix((v.astype(np.float64), (r, c)), shape=(n_rows, n_cols)).tocsr()   # duplicates summed
    g = BipartiteGraph(torch.from_numpy(r).cuda(), torch.from_numpy(c).cuda(), torch.from_numpy(v).cuda(), (n_rows, n_cols))
    return g, ref


# ------------------------------------------------------------------------------------------ graph
@pytest.mark.parametrize("shape_nnz", [((50, 70), 400), ((1, 1), 1), ((300, 200), 0), ((2000, 900), 60000)])
def test_csr_from_coo(shape_nnz):
    (m, n), nnz = shape_nnz
    g, ref = _graph(m, n, nnz, seed=nnz + m, heavy_rows=3 if nnz > 1000 else 0)
    got = g.fwd.to_scipy()
    got.sum_duplicates()
    assert abs(got - ref).max() < 1e-5 if nnz else got.nnz == 0
    got_t = g.bwd.to_scipy()
    got_t.sum_duplicates()
    assert abs(got_t - ref.T.tocsr()).max() < 1e-5 if nnz else got_t.nnz == 0
    # sorted by (row, col), rowptr monotone
    rp = g.fwd.rowptr.cpu().numpy()
    assert rp[0] == 0 and rp[-1] == nnz and (np.diff(rp) >= 0).all()
    if nnz > 1000:
        assert g.fwd.n_split_rows > 0   # the heavy rows went through the split plan


def test_row_normalize_matches_reference_formula():
    from mmssl_b200 import _lib
    from mmssl_b200._lib import ptr, stream
    from mmssl_b200.synthetic import csr_norm, make_bipartite
    r = make_bipartite(400, 150, 3000, seed=3)
    from mmssl_b200.graph import BipartiteGraph
    g = BipartiteGraph.from_scipy(r)
    lib = _lib.load(True)
    _lib.check(lib.mmssl_csr_row_normalize(ptr(g.fwd.rowptr), g.fwd.n_rows, ptr(g.fwd.vals), stream()))
    want = csr_norm(r)
    assert abs(g.fwd.to_scipy() - want).max() < 1e-6


# ------------------------------------------------------------------------------------------ spmm
@pytest.mark.parametrize("d", [64, 128, 256])
@pytest.mark.parametrize("nrhs", [1, 2, 3])
def test_spmm_plain(d, nrhs):
    from mmssl_b200 import ops
    g, ref = _graph(700, 500, 30000, seed=d + nrhs, heavy_rows=2)
    assert g.fwd.n_split_rows > 0
    torch.manual_seed(0)
    wide = torch.randn(500, nrhs * d + 8, device="cuda")
    xs = [wide[:, r * d:(r + 1) * d] for r in range(nrhs)]          # strided views (ld != d)
    ys = ops.spmm(g.fwd, xs)
    for x, y in zip(xs, ys):
        want = ref @ x.double().cpu().numpy()
        assert rel_err(y, torch.from_numpy(want)) < 2e-6
    # transposed operand
    xt = torch.randn(700, d, device="cuda")
    yt = ops.spmm(g.bwd, [xt])[0]
    assert rel_err(yt, torch.from_numpy(ref.T @ xt.double().cpu().numpy())) < 2e-6
    # launch twice: the split-row counters must have reset themselves
    yt2 = ops.spmm(g.bwd, [xt])[0]
    assert rel_err(yt2, yt) < 1e-6
    # rows up to 1024 non-zeros are reduced in a fixed order -> bitwise reproducible
    g2, _ = _graph(600, 500, 20000, seed=d, heavy_rows=40)     # ~170 nnz in each of 40 rows: split, not heavy
    assert g2.fwd.n_split_rows > 0
    y_a = ops.spmm(g2.fwd, [xs[0]])[0]
    y_b = ops.spmm(g2.fwd, [xs[0]])[0]
    assert torch.equal(y_a, y_b)


@pytest.mark.parametrize("impl", [2, 4, 6])
@pytest.mark.parametrize("nrhs", [1, 2, 3])
def test_spmm_impl_variants(impl, nrhs):
    """8-lane groups (impl bit 1) and 128-thread blocks (bit 2) give the same results as the default."""
    from mmssl_b200 import ops
    g, ref = _graph(900, 400, 40000, seed=11 + nrhs, heavy_rows=2)
    torch.manual_seed(0)
    xs = [torch.randn(400, 64, device="cuda") for _ in range(nrhs)]
    c = [torch.randn(900, 64, device="cuda") for _ in range(nrhs)]
    base = ops.spmm(g.fwd, xs, cs=c, alpha=0.5, epilogue=ops.EPI_SOFTMAX, impl=0)
    got = ops.spmm(g.fwd, xs, cs=c, alpha=0.5, epilogue=ops.EPI_SOFTMAX, impl=impl)
    for a, b in zip(base, got):
        assert rel_err(b, a) < 2e-6
    for x, y in zip(xs, ops.spmm(g.fwd, xs, impl=impl)):
        assert rel_err(y, torch.from_numpy(ref @ x.double().cpu().numpy())) < 2e-6


@pytest.mark.parametrize("d,nrhs", [(64, 1), (64, 3), (128, 2), (256, 1)])
def test_spmm_tma_hot_rows(d, nrhs):
    """TMA-staged hot-row variant (impl=1): same results as the LDG kernel, incl. epilogues and split rows."""
    from mmssl_b200 import ops
    rng = np.random.default_rng(d + nrhs)
    n_rows, n_cols, nnz = 3000, 5000, 90000
    pw = 1.0 / np.arange(1, n_cols + 1); pw /= pw.sum()                     # Zipf columns -> a real hot set
    r = rng.integers(0, n_rows, nnz); r[:20000] = rng.integers(0, 3, 20000)  # three heavy rows
    c = rng.choice(n_cols, nnz, p=pw)
    v = rng.standard_normal(nnz).astype(np.float32)
    ref = sp.coo_matrix((v.astype(np.float64), (r, c)), shape=(n_rows, n_cols)).tocsr()
    from mmssl_b200.graph import BipartiteGraph
    g = BipartiteGraph(torch.from_numpy(r).cuda(), torch.from_numpy(c).cuda(), torch.from_numpy(v).cuda(), (n_rows, n_cols))
    torch.manual_seed(0)
    xs = [torch.randn(n_cols, d, device="cuda") for _ in range(nrhs)]
    cs = [torch.randn(n_rows, d, device="cuda") for _ in range(nrhs)]
    ys = ops.spmm(g.fwd, xs, impl=ops.SPMM_IMPL_TMA)
    assert g.fwd.hot_edge_fraction > 0.3
    for x, y in zip(xs, ys):
        assert rel_err(y, torch.from_numpy(ref @ x.double().cpu().numpy())) < 1e-5
    a = ops.spmm(g.fwd, xs, cs=cs, alpha=0.5, epilogue=ops.EPI_SOFTMAX, impl=0)
    b = ops.spmm(g.fwd, xs, cs=cs, alpha=0.5, epilogue=ops.EPI_SOFTMAX, impl=ops.SPMM_IMPL_TMA)
    for u, w in zip(a, b):
        # the three heavy rows (~6.7k non-zeros, |logit| ~ 80) are reduced with float atomics in arrival order: an fp32 sum of
        # 6.7k terms moves by ~3e-4 between orders, and a softmax output by up to a quarter of that (measured on the earlier hardware: 1.1e-5 in
        # the suite, 7e-5 under compute-sanitizer's timing).  The plain products above are held to 1e-5.
        assert rel_err(w, u) < 2e-4
    yt = ops.spmm(g.bwd, [torch.randn(n_rows, d, device="cuda")], impl=ops.SPMM_IMPL_TMA)[0]   # A^T: hot set = heavy rows of A
    assert yt.shape == (n_cols, d) and torch.isfinite(yt).all()


def test_spmm_empty_and_tiny():
    from mmssl_b200 import ops
    from mmssl_b200.graph import BipartiteGraph
    e = torch.zeros(0, dtype=torch.int64, device="cuda")
    g = BipartiteGraph(e, e, torch.zeros(0, device="cuda"), (40, 30))
    x = torch.randn(30, 64, device="cuda")
    assert float(ops.spmm(g.fwd, [x])[0].abs().max()) == 0.0
    y = ops.spmm(g.fwd, [x], epilogue=ops.EPI_SOFTMAX)[0]          # softmax of an all-zero row = 1/d
    assert rel_err(y, torch.full((40, 64), 1 / 64)) < 1e-6


@pytest.mark.parametrize("d", [64, 128, 256])
def test_spmm_epilogues(d):
    from mmssl_b200 import ops
    g, ref = _graph(300, 260, 9000, seed=7 + d, heavy_rows=1)
    torch.manual_seed(1)
    x = torch.randn(260, d, device="cuda")
    c = torch.randn(300, d, device="cuda")
    base = torch.from_numpy(ref @ x.double().cpu().numpy())
    v = base + 0.25 * c.double().cpu()
    # + alpha*C then softmax, with running-sum init (mode 2) and accumulate (mode 1)
    sb = torch.randn(300, d, device="cuda")
    s = torch.empty(300, d, device="cuda")
    y = ops.spmm(g.fwd, [x], cs=[c], alpha=0.25, epilogue=ops.EPI_SOFTMAX, ss=[s], s_mode=2, sbases=[sb])[0]
    want = torch.softmax(v, dim=-1)
    # row 0 is a heavy row (3000 non-zeros: vector reductions in arrival order); its fp32 sum moves by ~1e-6 of its magnitude
    # (~50) from run to run and the softmax turns that into up to ~1e-5 (seen on hardware: 5e-6 .. 8e-6) -- hence 3e-5 here
    assert rel_err(y, want) < 3e-5
    assert rel_err(s, sb.double().cpu() + want) < 3e-5
    ops.spmm(g.fwd, [x], cs=[c], alpha=0.25, epilogue=ops.EPI_NONE, ss=[s], s_mode=1)
    assert rel_err(s, sb.double().cpu() + want + v) < 5e-6
    # softmax backward epilogue
    ysv = torch.softmax(torch.randn(300, d, device="cuda"), -1)
    t = ops.spmm(g.fwd, [x], cs=[c], alpha=0.25, epilogue=ops.EPI_SOFTMAX_BWD, ysaved=[ysv])[0]
    yd = ysv.double().cpu()
    assert rel_err(t, yd * (v - (v * yd).sum(-1, keepdim=True))) < 5e-6
    # in-place accumulate  y = y + A x
    acc = c.clone()
    ops.spmm(g.fwd, [x], [acc], cs=[acc], alpha=1.0)
    assert rel_err(acc, base + c.double().cpu()) < 5e-6


def test_spmm_function_autograd():
    from mmssl_b200.functional import spmm
    r, c, v = _rand_graph(120, 90, 1500, 5)
    a = torch.sparse_coo_tensor(torch.from_numpy(np.vstack([r, c])), torch.from_numpy(v), (120, 90)).cuda()
    x = torch.randn(90, 64, device="cuda", requires_grad=True)
    y = spmm(a, x)
    gy = torch.randn_like(y)
    y.backward(gy)
    xr = x.detach().cpu().double().requires_grad_(True)
    yr = torch.sparse.mm(a.cpu().double(), xr)
    yr.backward(gy.cpu().double())
    assert rel_err(y, yr) < 2e-6 and rel_err(x.grad, xr.grad) < 2e-6


# ------------------------------------------------------------------------------------------ dense
@pytest.mark.parametrize("ta,tb", [(False, False), (False, True), (True, False), (True, True)])
def test_sgemm(ta, tb):
    from mmssl_b200 import ops
    torch.manual_seed(2)
    m, n, k = 150, 70, 333
    a = torch.randn((k, m) if ta else (m, k), device="cuda")
    b = torch.randn((n, k) if tb else (k, n), device="cuda")
    out = torch.randn(m, n, device="cuda")
    c0 = out.clone()
    ops.sgemm(a, b, out, trans_a=ta, trans_b=tb, alpha=0.5, beta=2.0)
    A = a.double().cpu().t() if ta else a.double().cpu()
    B = b.double().cpu().t() if tb else b.double().cpu()
    assert rel_err(out, 0.5 * A @ B + 2.0 * c0.double().cpu()) < 1e-5
    out2 = c0.clone()
    ops.sgemm(a, b, out2, trans_a=ta, trans_b=tb, alpha=0.5, beta=1.0, split_k=4)
    assert rel_err(out2, 0.5 * A @ B + c0.double().cpu()) < 1e-5


@pytest.mark.parametrize("m,n,k", [(300, 64, 96), (7050, 64, 1024), (1000, 128, 520), (515, 256, 200), (4096, 64, 7050)])
def test_gemm_bf16x3_tensor_core(m, n, k):
    """wgmma projection GEMM vs fp64: the bf16 hi/lo split must deliver fp32-level accuracy."""
    from mmssl_b200 import ops
    torch.manual_seed(3)
    a = torch.randn(m, k, device="cuda")
    b = torch.randn(n, k, device="cuda") * 0.05
    a_hi, a_lo = ops.split_bf16(a)
    b_hi, b_lo = ops.split_bf16(b)
    floats, sk = ops.gemm_bf16x3_plan(m, n, k)
    part = torch.empty(floats, device="cuda")
    ops.gemm_bf16x3(a_hi, a_lo, b_hi, b_lo, m, n, k, sk, part)
    bias = torch.randn(n, device="cuda")
    mask = (torch.rand(m, n, device="cuda") > 0.2).float() / 0.8
    y = torch.empty(m, 2 * n, device="cuda")[:, n:]
    y_pre = torch.empty(m, n, device="cuda")
    ops.proj_epilogue(part, sk, m, n, bias, mask, y, y_pre)
    want = a.double().cpu() @ b.double().cpu().t() + bias.double().cpu()
    assert rel_err(y_pre, want) < 2e-5, rel_err(y_pre, want)
    assert rel_err(y, want * mask.double().cpu()) < 2e-5
    # weight-gradient epilogue = transposed reduction
    dw = torch.empty(n, m, device="cuda")
    ops.wgrad_epilogue(part, sk, m, n, dw)
    assert rel_err(dw, (a.double().cpu() @ b.double().cpu().t()).t()) < 2e-5


def test_split_bf16_transposed_with_mask():
    from mmssl_b200 import ops
    torch.manual_seed(4)
    x = torch.randn(77, 64, device="cuda")
    mask = (torch.rand(77, 64, device="cuda") > 0.5).float() * 2
    hi, lo = ops.split_bf16_t(x, mask)
    assert hi.shape == (64, 80)
    rec = (hi.float() + lo.float())[:, :77].t()
    assert rel_err(rec, (x * mask)) < 2e-5
    assert float(hi[:, 77:].float().abs().max()) == 0.0


# ------------------------------------------------------------------------------------------ row ops
@pytest.mark.parametrize("d", [64, 128, 256])
def test_rowops_vs_autograd(d):
    import torch.nn.functional as F
    from mmssl_b200 import ops
    torch.manual_seed(5)
    n = 203
    z = torch.randn(n, d); z[5] = 0          # a zero row exercises the eps clamp of F.normalize
    e, s, a, b = torch.randn(n, d), torch.randn(n, d), torch.randn(n, d), torch.randn(n, d)
    a[7] = 0
    g = torch.randn(n, d)
    zd, ed = z.double().requires_grad_(True), e.double()
    out_ref = ed + 0.36 * F.normalize(zd, dim=1)
    out_ref.backward(g.double())
    out, zn, nrm = ops.id_fuse_fwd(z.cuda(), e.cuda(), 0.36, torch.empty(n, d, device="cuda"))
    assert rel_err(out, out_ref) < 2e-6
    dz = ops.id_fuse_bwd(g.cuda(), zn, nrm, 0.36, torch.empty(n, d, device="cuda"))
    ok = torch.ones(n, dtype=torch.bool); ok[5] = False
    assert rel_err(dz[ok.cuda()], zd.grad[ok]) < 5e-6
    assert rel_err(dz[5], 0.36 * g[5].double() / 1e-12) < 1e-5      # clamp branch: g / eps
    # combine
    sd, ad, bd = s.double(), a.double().requires_grad_(True), b.double().requires_grad_(True)
    comb_ref = sd / 3 + 0.55 * F.normalize(ad, dim=1) + 0.55 * F.normalize(bd, dim=1)
    reg = 2e-3 * 0.5 * ((ad ** 2).sum() + (bd ** 2).sum())
    (comb_ref * g.double()).sum().add(reg).backward()
    comb, part = ops.combine_fwd(s.cuda(), a.cuda(), b.cuda(), 1 / 3, 0.55, torch.empty(n, d, device="cuda"))
    assert rel_err(comb, comb_ref) < 2e-6
    assert abs(float(part.sum()) - float((a ** 2).sum() + (b ** 2).sum())) < 1e-3 * float((a ** 2).sum())
    ext = torch.randn(n, d)
    ga, gb = torch.empty(n, d, device="cuda"), torch.empty(n, d, device="cuda")
    ops.combine_bwd(g.cuda(), a.cuda(), b.cuda(), ext.cuda(), None, 0.55, 2e-3, ga, gb)
    ok7 = torch.ones(n, dtype=torch.bool); ok7[7] = False
    assert rel_err(ga[ok7.cuda()], (ad.grad + ext.double())[ok7]) < 5e-6
    assert rel_err(gb, bd.grad) < 5e-6
    # softmax backward
    y = torch.softmax(torch.randn(n, d), -1)
    t = ops.softmax_bwd(y.cuda(), g.cuda(), 0.5, torch.empty(n, d, device="cuda"))
    yd, gd = y.double(), 0.5 * g.double()
    assert rel_err(t, yd * (gd - (gd * yd).sum(-1, keepdim=True))) < 5e-6


# ------------------------------------------------------------------------------------------ losses
@pytest.mark.parametrize("d", [64, 128])
def test_bpr_fused_and_autograd(d):
    from oracle import mmssl_oracle as O
    from mmssl_b200 import ops
    from mmssl_b200.functional import bpr_loss
    torch.manual_seed(6)
    U, I, B = 400, 300, 257
    uf, itf = torch.randn(U, d) * 0.3, torch.randn(I, d) * 0.3
    users = torch.randperm(U)[:B]; pos = torch.randint(0, I, (B,)); neg = torch.randint(0, I, (B,))
    cfg = O.HotPathConfig(embed_size=d, batch_size=1024)
    ufd, itd = uf.double().requires_grad_(True), itf.double().requires_grad_(True)
    mf, emb, _ = O.bpr_loss(ufd[users], itd[pos], itd[neg], cfg)
    (mf + emb).backward()
    # fused: table-level gradients with atomics
    g_u, g_i = torch.zeros(U, d, device="cuda"), torch.zeros(I, d, device="cuda")
    part, nb = ops.bpr(uf.cuda(), itf.cuda(), itf.cuda(), users.cuda(), pos.cuda(), neg.cuda(), mode=3,
                       reg_coef=cfg.emb_decay / cfg.batch_size, g_u=g_u, g_p=g_i, g_n=g_i)
    out5 = torch.empty(5, device="cuda")
    ops.loss_assemble(part, nb, B, cfg.emb_decay / cfg.batch_size, None, None, 0.0, None, None, 0, 0.0, out5)
    assert abs(float(out5[1]) - float(mf)) < 2e-6 and abs(float(out5[2]) - float(emb)) < 1e-9
    assert rel_err(g_u, ufd.grad) < 2e-5 and rel_err(g_i, itd.grad) < 2e-5
    # three-tensor autograd signature (main.py:499-511)
    ub, pb, nb_ = (t.cuda().requires_grad_(True) for t in (uf[users], itf[pos], itf[neg]))
    mf2, emb2, reg2 = bpr_loss(ub, pb, nb_, decay=cfg.emb_decay, batch_size=cfg.batch_size)
    (2.0 * mf2 + 3.0 * emb2).backward()
    ubd, pbd, nbd = (t.double().requires_grad_(True) for t in (uf[users], itf[pos], itf[neg]))
    mfr, embr, _ = O.bpr_loss(ubd, pbd, nbd, cfg)
    (2.0 * mfr + 3.0 * embr).backward()
    assert reg2 == 0.0 and abs(float(mf2) - float(mfr)) < 2e-6
    for got, want in ((ub.grad, ubd.grad), (pb.grad, pbd.grad), (nb_.grad, nbd.grad)):
        assert rel_err(got, want) < 2e-5


@pytest.mark.parametrize("n,d", [(64, 64), (257, 64), (1024, 64), (130, 128), (96, 256)])
def test_infonce_forward_backward(n, d):
    from oracle import mmssl_oracle as O
    from mmssl_b200.functional import batched_contrastive_loss
    torch.manual_seed(7)
    z1, z2 = torch.randn(n, d), torch.randn(n, d) * 0.5
    z1[3] = 0        # zero row: normalize eps path
    cfg = O.HotPathConfig(embed_size=d)
    a, b = z1.double().requires_grad_(True), z2.double().requires_grad_(True)
    want = O.infonce(a, b, cfg)
    (1.7 * want).backward()
    x1, x2 = z1.cuda().requires_grad_(True), z2.cuda().requires_grad_(True)
    got = batched_contrastive_loss(x1, x2, tau=cfg.tau)
    (1.7 * got).backward()
    assert abs(float(got) - float(want)) < 1e-5 * abs(float(want))
    ok = torch.ones(n, dtype=torch.bool); ok[3] = False
    assert rel_err(x1.grad[ok.cuda()], a.grad[ok]) < 5e-5
    assert rel_err(x2.grad, b.grad) < 5e-5


def test_feat_reg_autograd():
    from mmssl_b200.functional import feat_reg_loss
    torch.manual_seed(8)
    ts = [torch.randn(r, 64) for r in (150, 150, 333, 333)]
    cu = [t.cuda().requires_grad_(True) for t in ts]
    loss = feat_reg_loss(*cu, n_items=150, feat_reg_decay=1e-5)
    (loss * 4.0).backward()
    td = [t.double().requires_grad_(True) for t in ts]
    want = 1e-5 * sum(0.5 * (t ** 2).sum() for t in td) / 150
    (want * 4.0).backward()
    assert abs(float(loss) - float(want)) < 1e-6 * float(want) + 1e-12
    for g, w in zip(cu, td):
        assert rel_err(g.grad, w.grad) < 1e-5


def test_adamw_matches_torch():
    from mmssl_b200 import ops
    torch.manual_seed(9)
    shapes = [(1000, 64), (64,), (64, 130), (7,)]
    ps = [torch.randn(s) for s in shapes]
    ref = [p.clone().requires_grad_(True) for p in ps]
    opt = torch.optim.AdamW(ref, lr=5.5e-4)
    cu = [p.cuda() for p in ps]
    m = [torch.zeros_like(p) for p in cu]; v = [torch.zeros_like(p) for p in cu]
    step = torch.zeros(1, dtype=torch.int32, device="cuda")
    for _ in range(3):
        gs = [torch.randn(s) for s in shapes]
        for r, g in zip(ref, gs):
            r.grad = g.clone()
        opt.step()
        ops.step_tick(step)
        ops.adamw(cu, [g.cuda() for g in gs], m, v, step, 5.5e-4)
    for c, r in zip(cu, ref):
        assert rel_err(c, r) < 2e-6


def test_dropout_mask_from_ones_matches_torch_stream():
    """Models.MMSSL draws its dropout masks as dropout(ones): same Philox consumption as the
    reference's dropout(x) on an [I, d] tensor."""
    import torch.nn.functional as F
    x = torch.randn(7050, 64, device="cuda")
    torch.manual_seed(123); a = F.dropout(x, 0.2, True)
    torch.manual_seed(123); m = F.dropout(torch.ones_like(x), 0.2, True)
    assert torch.equal(a, x * m)


def test_device_triple_sampler_semantics():
    """GPU sampler vs the semantics of Data.sample (load_data.py:153-191)."""
    from mmssl_b200.sampler import DeviceTripleSampler
    from mmssl_b200.synthetic import make_dataset
    ds = make_dataset("tiktok")
    smp = DeviceTripleSampler(ds.train, seed=7)
    dense_row = lambda u: set(ds.train.indices[ds.train.indptr[u]:ds.train.indptr[u + 1]].tolist())
    out = torch.empty(3, 1024, dtype=torch.int64, device="cuda")
    step = torch.zeros(1, dtype=torch.int32, device="cuda")
    seen_users, pos_hits = [], 0
    batches = []
    for s in range(20):
        step.fill_(s)
        smp.sample_into(out, step_dev=step)
        u, p, n = (t.cpu().numpy() for t in out)
        batches.append((u.copy(), p.copy(), n.copy()))
        assert len(set(u.tolist())) == 1024                                    # distinct users
        assert (np.diff(ds.train.indptr)[u] > 0).all()                         # users with >= 1 item
        for k in range(0, 1024, 37):
            row = dense_row(int(u[k]))
            assert int(p[k]) in row and int(n[k]) not in row
        seen_users.append(u)
    assert int((smp.claim != 0x7fffffff).sum()) == 0                           # claim table left clean
    # deterministic in (seed, step); different steps differ
    step.fill_(3)
    smp.sample_into(out, step_dev=step)
    assert np.array_equal(out[0].cpu().numpy(), batches[3][0]) and np.array_equal(out[2].cpu().numpy(), batches[3][2])
    assert not np.array_equal(batches[3][0], batches[4][0])
    # roughly uniform over users: every user should be hit about 20*1024/U times
    cnt = np.bincount(np.concatenate(seen_users), minlength=ds.n_users)
    exp = 20 * 1024 / ds.n_users
    assert abs(cnt.mean() - exp) < 1e-9 and cnt.max() < exp * 5 + 10
