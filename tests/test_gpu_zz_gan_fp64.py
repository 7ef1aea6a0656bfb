"""The GAN side (csrc/gan.cu, the GEMM routes, mmssl_b200/gan.py) against float64, at the shapes and values where fp32
kernels go wrong: one- and two-column BatchNorms, ragged widths, constant and fully dropped columns, a column whose mean is
1e3 times its spread, saturated sigmoid heads, zero-norm penalty rows, users whose training row covers every item.

Inputs are float64 draws rounded to fp32.  The yardstick is the reference's own expression (torch autograd, oracle/gan_oracle.py)
evaluated in float64 on those inputs; where only a closed form exists it is the closed form in float64 (pinned to autograd at
1e-9 in tests/test_gan_oracle.py).  A device result may be at most 4x as far from float64 as the fp32 evaluation of the same
expression on the same inputs, and never has to be closer than fullstep_check.FP64_FLOOR (within_fp32_reach).  The same
bodies run on the CPU under the cuemu emulator at small sizes (tests/test_emu_gan_fp64.py)."""
import zlib

import numpy as np
import pytest
import scipy.sparse as sp
import torch
import torch.nn.functional as F

from oracle import gan_oracle as GO
from tests import gan_ops_cpu as REF
from tests.fullstep_check import FP64_FLOOR, d_step_vs_float64, within_fp32_reach

pytestmark = pytest.mark.gpu
FLOOR = 1e-5                                    # single kernels: no GEMM in between
EPS = 1e-5


def _gen(*key):
    return torch.Generator().manual_seed(zlib.crc32(repr(key).encode()))


def _r(x):
    """float64 draw -> the fp32 value the device gets, back in float64 (the point where both references are evaluated)."""
    return x.float().double()


def _cuda(*ts):
    return [t.float().cuda() for t in ts]


def _check(got, want64, ref32, what, floor=FLOOR):
    assert bool(torch.isfinite(got.cpu()).all()), f"{what}: non-finite device result"
    return within_fp32_reach(got.cpu(), want64, ref32, floor, what)


def _both(fn, *args):
    """fn evaluated in float64 and in float32 on the same (fp32-representable) inputs."""
    to = lambda dt: [a.to(dt) if torch.is_tensor(a) and a.is_floating_point() else a for a in args]
    return fn(*to(torch.float64)), fn(*to(torch.float32))


# ------------------------------------------------------------------------------------------ BatchNorm column ops
BN_H = [1, 2, 3, 5, 12, 25, 881, 1762]
BN_N = [2, 3, 48, 2048, 32768]


def _bn_inputs(n, h, seed=0):
    g = _gen("bn", n, h, seed)
    a = torch.randn(n, h, generator=g, dtype=torch.float64) * 3 + 1
    mask = ((torch.rand(n, h, generator=g, dtype=torch.float64) >= 0.31) / 0.69)
    a[:, 0] = 0.7                                               # constant column: var = 0, rstd = eps^-1/2
    if h > 1:
        mask[:, 1] = 0.0                                        # dropped in every row
    if h > 2:
        a[:, 2] = 1e3 + torch.randn(n, generator=g, dtype=torch.float64)    # mean = 1e3 x std
    bias = torch.randn(h, generator=g, dtype=torch.float64) * 0.1
    gamma = 1 + 0.2 * torch.randn(h, generator=g, dtype=torch.float64)
    beta = 0.1 * torch.randn(h, generator=g, dtype=torch.float64)
    rm, rv = torch.randn(h, generator=g, dtype=torch.float64), torch.rand(h, generator=g, dtype=torch.float64) + 0.5
    return [_r(t) for t in (a, bias, gamma, beta, mask, rm, rv)], g


def _bn_ref(a, bias, gamma, beta, mask, rm, rv):
    """The reference's layer: BatchNorm1d (training mode) of (a + bias), dropout mask; running statistics updated in place."""
    rm, rv = rm.clone(), rv.clone()
    h = F.batch_norm(a + bias, rm, rv, gamma, beta, True, 0.1, EPS) * mask
    mu, var = a.mean(0), a.var(0, unbiased=False)
    r = (var + EPS).rsqrt()
    return h, (a - mu) * r, r, rm, rv


def check_bn_ops(n, h):
    from mmssl_b200 import gan_ops as K
    (a, bias, gamma, beta, mask, rm, rv), g = _bn_inputs(n, h)
    hi, lo = _both(_bn_ref, a, bias, gamma, beta, mask, rm, rv)
    rm_d, rv_d = _cuda(rm, rv)
    got = K.bn_fwd(*_cuda(a, bias, gamma, beta, mask), rm_d, rv_d)
    for j, name in enumerate(("h", "ah", "rstd")):
        _check(got[j], hi[j], lo[j], f"bn_fwd {name} n={n} h={h}")
    _check(rm_d, hi[3], lo[3], f"bn_fwd running_mean n={n} h={h}")
    _check(rv_d, hi[4], lo[4], f"bn_fwd running_var n={n} h={h}")
    ah, r = _r(hi[1]), _r(hi[2])

    # bn_bwd: d/d(a, gamma, beta) of sum(dh * h) through F.batch_norm
    dh = _r(torch.randn(n, h, generator=g, dtype=torch.float64))

    def bwd(a, gamma, beta, mask, dh):
        a, gamma, beta = (t.clone().requires_grad_(True) for t in (a, gamma, beta))
        y = F.batch_norm(a, None, None, gamma, beta, True, 0.1, EPS) * mask
        return torch.autograd.grad((y * dh).sum(), (a, gamma, beta))
    hi, lo = _both(bwd, a, gamma, beta, mask, dh)
    da, dy, dg, db = K.bn_bwd(*_cuda(dh, mask, gamma, ah, r))
    for got_, j, name in ((da, 0, "da"), (dg, 1, "dgamma"), (db, 2, "dbeta")):
        _check(got_, hi[j], lo[j], f"bn_bwd {name} n={n} h={h}")
    assert torch.equal(dy.cpu(), dh.float() * mask.float())

    # gp_rev_bn: adjoint of da = bn_bwd(dh, ah, r, gamma) seeded with q (closed form, differentiated by autograd)
    q = _r(torch.randn(n, h, generator=g, dtype=torch.float64))

    def rev(dh, ah, r, gamma, mask, q):
        dh, ah, r, gamma = (t.clone().requires_grad_(True) for t in (dh, ah, r, gamma))
        return torch.autograd.grad((q * REF.bn_bwd(dh, mask, gamma, ah, r)[0]).sum(), (dh, ah, r, gamma))
    hi, lo = _both(rev, dh, ah, r, gamma, mask, q)
    got = K.gp_rev_bn(*_cuda(q, _r(dh.float() * mask.float()), ah, r, gamma, mask))
    for j, name in enumerate(("dh_bar", "ah_bar", "r_bar", "g_gamma")):
        _check(got[j], hi[j], lo[j], f"gp_rev_bn {name} n={n} h={h}")

    # bn_fwd_rev: adjoint of a -> (h, ah, r) with extra adjoints of ah and r
    h_bar, ah_bar = (_r(torch.randn(n, h, generator=g, dtype=torch.float64)) for _ in range(2))
    r_bar = _r(torch.randn(h, generator=g, dtype=torch.float64))

    def fwd_rev(a, gamma, beta, mask, h_bar, ah_bar, r_bar):
        a, gamma, beta = (t.clone().requires_grad_(True) for t in (a, gamma, beta))
        mu, var = a.mean(0), a.var(0, unbiased=False)
        rr = (var + EPS).rsqrt()
        x = (a - mu) * rr
        hh = (x * gamma + beta) * mask
        return torch.autograd.grad((h_bar * hh).sum() + (ah_bar * x).sum() + (r_bar * rr).sum(), (a, gamma, beta))
    hi, lo = _both(fwd_rev, a, gamma, beta, mask, h_bar, ah_bar, r_bar)
    got = K.bn_fwd_rev(*_cuda(h_bar, mask, gamma, ah, r, ah_bar, r_bar))
    for j, name in enumerate(("a_bar", "g_gamma", "g_beta")):
        _check(got[j], hi[j], lo[j], f"bn_fwd_rev {name} n={n} h={h}")

    # colsum adds n / 32 terms in sequence per row lane: its own rounding bound is that many fp32 half-ulps
    hi, lo = _both(lambda x: x.sum(0), a)
    _check(K.colsum(*_cuda(a)), hi, lo, f"colsum n={n} h={h}", max(FLOOR, -(-n // 32) * 2.0 ** -24))


@pytest.mark.parametrize("n,h", [(n, h) for n in BN_N for h in BN_H if n * h <= 2 ** 25])     # n = 32768: h up to 881
def test_bn_ops_vs_float64(n, h):
    check_bn_ops(n, h)


# ------------------------------------------------------------------------------------------ sigmoid head
def _head_inputs(n, h, sat):
    g = _gen("head", n, h, sat)
    h2 = _r(torch.randn(n, h, generator=g, dtype=torch.float64))
    w3 = _r(torch.randn(1, h, generator=g, dtype=torch.float64) * 0.2)
    z0 = h2 @ w3.view(-1)
    shift = {"none": 0.0, "high": 25.0 + float(z0.abs().max()), "low": -95.0 - float(z0.abs().max())}.get(sat, 0.0)
    b3 = _r(torch.full((1,), shift, dtype=torch.float64))
    if sat == "half":                          # every other row pushed past z = 20 through one column of h2
        h2[::2, 0] = float(np.float32((25.0 + float(z0.abs().max())) / float(w3[0, 0])))
    return h2, w3, b3, g


def check_head_ops(n, h, sat):
    from mmssl_b200 import gan_ops as K
    h2, w3, b3, g = _head_inputs(n, h, sat)

    def fwd(h2, w3, b3):
        s = torch.sigmoid(h2 @ w3.view(-1) + b3)
        return s, s.sum().view(1)
    hi, lo = _both(fwd, h2, w3, b3)
    s_d, ssum_d = K.head_fwd(*_cuda(h2, w3, b3))
    _check(s_d, hi[0], lo[0], f"head_fwd s n={n} h={h} {sat}")
    _check(ssum_d, hi[1], lo[1], f"head_fwd sum n={n} h={h} {sat}")
    s = _r(hi[0])
    if sat == "high":
        assert bool((s_d.cpu() == 1).all())
    coef = -1.0 / n

    def bwd(h2, w3, b3):                       # d/d(h2, w3, b3) of coef * 100 * sum(sigmoid(z)), and d/dz
        h2, w3, b3 = (t.clone().requires_grad_(True) for t in (h2, w3, b3))
        z = h2 @ w3.view(-1) + b3
        z.retain_grad()
        (coef * 100 * torch.sigmoid(z).sum()).backward()
        return h2.grad, z.grad, w3.grad.view(-1), b3.grad
    hi, lo = _both(bwd, h2, w3, b3)
    got = K.head_bwd(s.float().cuda(), coef, *_cuda(w3, h2))
    for j, name in enumerate(("dh2", "dz", "dw3", "db3")):
        if sat == "high":                      # s == 1 in fp32: the reference's fp32 arithmetic gives exactly 0
            assert float(got[j].abs().max()) == 0.0 and float(lo[j].abs().max()) == 0.0, name
        else:
            _check(got[j].view_as(hi[j]), hi[j], lo[j], f"head_bwd {name} n={n} h={h} {sat}")

    # gp_head_rev: adjoint of [z -> dz = 100 s (1 - s) (coef 1) -> dh2 = dz (x) w3] and of the forward z = h2 w3 + b3
    dh2_bar = _r(torch.randn(n, h, generator=g, dtype=torch.float64))
    dz = _r(100 * s * (1 - s))

    def rev(h2, w3, b3, dh2_bar):
        h2, w3, b3 = (t.clone().requires_grad_(True) for t in (h2, w3, b3))
        sg = torch.sigmoid(h2 @ w3.view(-1) + b3)
        dzz = 100 * sg * (1 - sg)
        return torch.autograd.grad((dh2_bar * (dzz.unsqueeze(1) * w3.view(1, -1))).sum(), (h2, w3, b3))
    hi, lo = _both(rev, h2, w3, b3, dh2_bar)
    h_bar, g_w3, g_b3 = K.gp_head_rev(*_cuda(dh2_bar, dz, s, w3, h2))
    for got_, j, name in ((h_bar, 0, "h_bar"), (g_w3, 1, "g_w3"), (g_b3, 2, "g_b3")):
        if sat == "high":
            assert float(got_.abs().max()) == 0.0 and float(lo[j].abs().max()) == 0.0, name
        else:
            _check(got_.view_as(hi[j]), hi[j], lo[j], f"gp_head_rev {name} n={n} h={h} {sat}")


@pytest.mark.parametrize("sat", ["none", "high", "low", "half"])
@pytest.mark.parametrize("n,h", [(48, 1), (2048, 5), (2048, 881), (3, 5)])
def test_head_ops_vs_float64(n, h, sat):
    check_head_ops(n, h, sat)


# ------------------------------------------------------------------------------------------ penalty rows
def check_gp_rows(n, w):
    from mmssl_b200 import gan_ops as K
    g = _gen("gp", n, w)
    gx = torch.randn(n, w, generator=g, dtype=torch.float64) * (2.0 / w ** 0.5)
    gx[0] = 0.0                                                   # norm 0: zero gradient, adds 1 to the penalty
    gx[1] = 0.0
    gx[1, w // 2] = 1.0                                           # norm exactly 1
    gx[2] = 1e-20 * torch.randn(w, generator=g, dtype=torch.float64)
    gx[3] = 0.0
    gx = _r(gx)

    def ref(gx):
        ga = gx.clone().requires_grad_(True)
        gp = 0.3 * ((ga.norm(2, dim=1) - 1) ** 2).mean()
        return gp.detach().view(1), torch.autograd.grad(gp, ga)[0]
    hi, lo = _both(ref, gx)
    gp, gbar = K.gp_rows(gx.float().cuda(), 0.3)
    _check(gp, hi[0], lo[0], f"gp_rows gp n={n} w={w}")
    _check(gbar, hi[1], lo[1], f"gp_rows gbar n={n} w={w}")
    gb = gbar.cpu()
    assert float(gb[0].abs().max()) == 0.0 and float(gb[1].abs().max()) == 0.0 and float(gb[3].abs().max()) == 0.0


@pytest.mark.parametrize("w", [1, 7, 7050, 18357])
@pytest.mark.parametrize("n", [5, 64])
def test_gp_rows_vs_float64(n, w):
    check_gp_rows(n, w)


# ------------------------------------------------------------------------------------------ u_sim and the real rows
def _csr_with_edge_users(U, I, seed):
    R = sp.random(U, I, density=min(0.2, 20.0 / I), format="lil", random_state=seed, dtype=np.float32)
    R[0, :] = 1.0                                                 # user 0: every item is a training item
    R[1, :] = 0.0                                                 # user 1: no training item
    R = R.tocsr()
    R.data[:] = 1.0
    R.sort_indices()
    return R


def check_usim_and_real_rows(U, I, B, d):
    from mmssl_b200 import gan_ops as K
    g = _gen("usim", U, I, B, d)
    R = _csr_with_edge_users(U, I, 3)
    indptr, indices = torch.from_numpy(R.indptr.astype(np.int64)), torch.from_numpy(R.indices.astype(np.int64))
    users = torch.cat((torch.tensor([0, 1]), torch.randperm(U - 2, generator=g)[:B - 2] + 2))
    dev = [t.cuda() for t in (users, indptr, indices)]
    keep = 1 - torch.from_numpy(np.asarray(R[users.tolist()].todense())).double()
    scores = _r(torch.randn(B, I, generator=g, dtype=torch.float64))

    def fin(scores):
        raw = scores * keep.to(scores.dtype)
        return F.normalize(raw, p=2, dim=1), raw.norm(2, dim=1).clamp_min(1e-12)
    hi, lo = _both(fin, scores)
    y, nrm = K.usim_finish(scores.float().cuda(), *dev)
    _check(y, hi[0], lo[0], f"usim_finish y I={I}")
    _check(nrm, hi[1], lo[1], f"usim_finish nrm I={I}")
    assert float(y.cpu()[0].abs().max()) == 0.0 and float(nrm.cpu()[0]) == np.float32(1e-12)

    go = _r(torch.randn(B, I, generator=g, dtype=torch.float64))

    def bwd(scores, go):                                          # d/d scores of sum(go * F.normalize(scores * keep))
        sc = scores.clone().requires_grad_(True)
        return torch.autograd.grad((go * F.normalize(sc * keep.to(sc.dtype), p=2, dim=1)).sum(), sc)[0]
    hi_b, lo_b = _both(bwd, scores, go)
    got = K.usim_bwd_pre(*_cuda(go, _r(hi[0]), _r(hi[1])), *dev)
    _check(got, hi_b, lo_b, f"usim_bwd_pre I={I}")

    uni = torch.rand(B, I, generator=g, dtype=torch.float64)
    uni[:, 0] = 0.0                                               # the two ends of torch.rand's fp32 range
    uni[:, 1] = 1.0 - 2.0 ** -24
    uni = _r(uni)
    ui = _r(hi[0])
    cfg = GO.GanConfig()
    hi, lo = _both(lambda u, s: GO.real_rows(users.tolist(), R, u, s, cfg), uni, ui)
    got = K.real_rows(*dev, *_cuda(uni, ui), cfg.log_log_scale, cfg.real_data_tau, cfg.ui_pre_scale)
    _check(got, hi, lo, f"real_rows I={I}")


@pytest.mark.parametrize("U,I,B,d", [(120, 97, 32, 64), (19445, 7050, 1024, 64), (300, 7050, 7, 32)])
def test_usim_and_real_rows_vs_float64(U, I, B, d):
    check_usim_and_real_rows(U, I, B, d)


# ------------------------------------------------------------------------------------------ elementwise and row movement
def check_elementwise(n, w):
    from mmssl_b200 import gan_ops as K
    g = _gen("elem", n, w)
    alpha = _r(torch.rand(n, generator=g, dtype=torch.float64))
    alpha[0], alpha[-1] = 0.0, 1.0 - 2.0 ** -24
    xr, xf = (_r(torch.randn(n, w, generator=g, dtype=torch.float64)) for _ in range(2))
    hi, lo = _both(lambda a, r, f: a.view(-1, 1) * r + (1 - a.view(-1, 1)) * f, alpha, xr, xf)
    _check(K.interpolate(*_cuda(alpha, xr, xf)), hi, lo, f"interpolate n={n} w={w}")
    acc = xr.float().cuda()
    K.add_scaled(acc, xf.float().cuda(), -0.7)
    hi, lo = _both(lambda r, f: r + (-0.7) * f, xr, xf)
    _check(acc, hi, lo, f"add_scaled n={n} w={w}")
    table = _r(torch.randn(n + 3, w, generator=g, dtype=torch.float64))
    rows = torch.randint(0, n + 3, (2 * n,), generator=g)
    rows[: n // 2 + 1] = rows[0]                                  # one id many times over
    assert torch.equal(K.gather_rows(table.float().cuda(), rows.cuda()).cpu(), table.float()[rows])
    src = _r(torch.randn(2 * n, w, generator=g, dtype=torch.float64))
    dst = table.float().cuda()
    K.scatter_add_rows(dst, rows.cuda(), src.float().cuda())

    def sc(t, s):
        return t.clone().index_add_(0, rows, s)
    hi, lo = _both(sc, table, src)
    _check(dst, hi, lo, f"scatter_add_rows n={n} w={w}")


@pytest.mark.parametrize("n,w", [(2, 1), (7, 33), (64, 97), (2048, 7050), (5, 18357)])
def test_elementwise_vs_float64(n, w):
    check_elementwise(n, w)


# ------------------------------------------------------------------------------------------ the composite D step and G side
def random_d_state(I, g, sat="none"):
    """A Discriminator state (kaiming-like weights, non-trivial BatchNorm affine).  sat="all": net.8.bias = +30, every head
    saturates in fp32.  sat="half": one input column routed straight to the head, so that rows whose column-0 entry is high
    have z around 60 (saturated) and the others around 0."""
    h1, h2 = I // 4, I // 8
    kn = lambda o, i: torch.randn(o, i, generator=g, dtype=torch.float64) * (2.0 / i) ** 0.5
    S = {"net.0.weight": kn(h1, I), "net.0.bias": 0.1 * torch.randn(h1, generator=g, dtype=torch.float64),
         "net.2.weight": 1 + 0.2 * torch.randn(h1, generator=g, dtype=torch.float64),
         "net.2.bias": 0.1 * torch.randn(h1, generator=g, dtype=torch.float64),
         "net.4.weight": kn(h2, h1), "net.4.bias": 0.1 * torch.randn(h2, generator=g, dtype=torch.float64),
         "net.6.weight": 1 + 0.2 * torch.randn(h2, generator=g, dtype=torch.float64),
         "net.6.bias": 0.1 * torch.randn(h2, generator=g, dtype=torch.float64),
         "net.8.weight": kn(1, h2), "net.8.bias": torch.zeros(1, dtype=torch.float64)}
    if sat == "all":
        S["net.8.bias"].fill_(30.0)
    elif sat == "half":
        S["net.0.weight"][0] = 0.0
        S["net.0.weight"][0, 0] = 50.0
        S["net.4.weight"][0] = 0.0
        S["net.4.weight"][0, 0] = 1.0
        for k in ("net.2", "net.6"):
            S[k + ".weight"][0], S[k + ".bias"][0] = 1.0, 0.0
        S["net.8.weight"] *= 0.1
        S["net.8.weight"][0, 0] = 30.0
        S["net.8.bias"].fill_(30.0)
    S = {k: _r(v).float() for k, v in S.items()}
    for k, n in (("net.2", h1), ("net.6", h2)):
        S[k + ".running_mean"], S[k + ".running_var"] = torch.zeros(n), torch.ones(n)
        S[k + ".num_batches_tracked"] = torch.zeros((), dtype=torch.int64)
    return S


def composite_check(I, d, B, route, sat="none", seed=0):
    """gan.d_step (penalty included) and gan.g_side on the device from one state, with no optimiser step between them,
    against the float64 autograd of the reference's D step and G_rate * G_lossf term on the same state, rows and draws."""
    from mmssl_b200 import gan, gan_ops as K
    g = _gen("composite", I, d, B, sat, seed)
    U = max(3 * B, 40)
    R = _csr_with_edge_users(U, I, seed)
    indptr, indices = torch.from_numpy(R.indptr.astype(np.int64)), torch.from_numpy(R.indices.astype(np.int64))
    users = torch.randperm(U, generator=g)[:B]
    dev = [t.cuda() for t in (users, indptr, indices)]
    S = random_d_state(I, g, sat)
    h1, h2 = I // 4, I // 8
    tables = [_r(torch.randn(n, d, generator=g, dtype=torch.float64)).float() for n in (U, I, U, I, U, I)]
    mk = lambda w, p: ((torch.rand(2 * B, w, generator=g) >= p) / (1 - p)).float()
    m1, m2 = [mk(h1, 0.31) for _ in range(4)], [mk(h2, 0.5) for _ in range(4)]
    gu, al = torch.rand(B, I, generator=g), torch.rand(2 * B, generator=g)
    floor = FP64_FLOOR[route]
    old = K.GEMM_IMPL
    K.GEMM_IMPL = route
    try:
        tc = [t.cuda() for t in tables]
        cs = [gan.u_sim_forward(K, tc[2 * j], tc[2 * j + 1], *dev) for j in range(3)]       # ui, image, text
        if sat == "half":          # column 0 high on every other user, in the fake, real and penalty rows alike
            for c in cs:
                y = c["y"]
                y[:, 0] = 0.0
                y[::2, 0] = 0.5
        for j, c in enumerate(cs if sat != "half" else ()):
            hi, lo = _both(lambda uf, itf: GO.u_sim(users.tolist(), uf, itf, R, B), tables[2 * j], tables[2 * j + 1])
            within_fp32_reach(c["y"].cpu(), hi, lo, floor, f"u_sim {j} I={I} d={d} B={B} {route}")
        ui, img, txt = (c["y"] for c in cs)
        D = gan.DiscriminatorState({k: v.clone().cuda() for k, v in S.items()})
        K.weights_changed()
        K.register_weights([D.t["net.0.weight"], D.t["net.4.weight"]])
        hp = gan.GanHyper()
        dres = gan.d_step(K, D, hp, img, txt, ui, *dev, gu.cuda(), al.cuda(), [m.cuda() for m in m1[:3]], [m.cuda() for m in m2[:3]])
        # no optimiser step between the two sides: the G side sees the state the D step started from
        for k in gan.PARAMS:
            D.t[k].copy_(S[k].cuda())
        K.weights_changed()
        s_sum, dx_img, dx_txt = gan.g_side(K, D, hp, cs[1], cs[2], m1[3].cuda(), m2[3].cuda())
        for k in gan.PARAMS + ("gp", "lossf_sum", "lossr_sum"):
            v = dres["grads"][k] if k in gan.PARAMS else dres[k]
            assert bool(torch.isfinite(v.cpu()).all()), (k, "not finite")
        gcfg = GO.GanConfig()
        if sat == "half":          # the state does what it is for: some heads of the fake call saturate in fp32, not all
            out = GO.discriminator(torch.cat((img, txt)).cpu(), {k: v.clone() for k, v in S.items()}, m1[0], m2[0])
            assert 0 < int((out == 100).sum()) < out.numel(), int((out == 100).sum())
        if sat == "all":         # fp32 gives s == 1 on every row: the reference's own arithmetic is the yardstick
            rr = GO.real_rows(users.tolist(), R, gu, ui.cpu(), gcfg)
            lo = GO.d_step_grads(S, torch.cat((img, txt)).cpu(), torch.cat((rr, rr)), al, m1[:3], m2[:3], gcfg)
            assert float(lo["gp"]) == pytest.approx(hp.gp_lambda, rel=1e-6)
            assert abs(float(dres["gp"].cpu()) - hp.gp_lambda) <= 2e-7 * hp.gp_lambda, float(dres["gp"].cpu())
            for k in gan.PARAMS:
                got = dres["grads"][k].cpu().view_as(lo["grads"][k])
                assert torch.equal(got, lo["grads"][k]) and float(got.abs().max()) == 0.0, k
            assert float(dx_img.abs().max()) == 0.0 and float(dx_txt.abs().max()) == 0.0
            assert float(dres["lossf_sum"].cpu()) == 2 * B and float(s_sum.cpu()) == 2 * B
            return None
        dist = d_step_vs_float64(S, dres, ui, img, txt, users, R, gu, al, m1, m2, gcfg, floor,
                                 what=f"I={I} d={d} B={B} {route} {sat}")
        res = {dt: GO.g_side_grads({k: v.to(dt) if v.is_floating_point() else v for k, v in S.items()}, img.cpu(), txt.cpu(),
                                   m1[3], m2[3], gcfg) for dt in (torch.float64, torch.float32)}
        hi, lo = res[torch.float64], res[torch.float32]
        dist["G s_sum"] = within_fp32_reach(s_sum.cpu() * 100.0, hi[0].sum().view(1), lo[0].sum().view(1), floor, "G s_sum")
        dist["G dx_image"] = within_fp32_reach(dx_img.cpu(), hi[1], lo[1], floor, f"I={I} d={d} B={B} {route} G dx image")
        dist["G dx_text"] = within_fp32_reach(dx_txt.cpu(), hi[2], lo[2], floor, f"I={I} d={d} B={B} {route} G dx text")
        return dist
    finally:
        K.GEMM_IMPL = old
        K.weights_changed()


COMPOSITE = [(8, 32, 2), (9, 64, 24), (15, 96, 24), (16, 128, 24), (97, 96, 24), (101, 192, 24), (103, 256, 24),
             (97, 64, 2), (97, 256, 1024), (7050, 64, 1024)]


@pytest.mark.parametrize("route", ["simt", "tc"])
@pytest.mark.parametrize("I,d,B", COMPOSITE)
def test_d_step_and_g_side_vs_float64(I, d, B, route):
    dist = composite_check(I, d, B, route)
    print(f"I={I} d={d} B={B} {route}: distance to float64 (device, fp32 autograd):",
          {k: ("%.3g" % a, "%.3g" % b) for k, (a, b) in dist.items()})


@pytest.mark.parametrize("route", ["simt", "tc"])
@pytest.mark.parametrize("sat", ["all", "half"])
def test_d_step_saturated_heads(sat, route):
    composite_check(97, 64, 24, route, sat=sat)


def full_step_from_saturated_state(dev):
    """One FullStep iteration from a Discriminator whose heads all saturate (net.8.bias = +30): the penalty rows have norm 0,
    the reference carries on with gp = lambda and zero penalty gradients; every parameter must stay finite."""
    from tests import fullstep_check
    z, c = fullstep_check.load_trace()
    fs, P, t = fullstep_check.build(z, c, dev)
    fs.D.t["net.8.bias"].fill_(30.0)
    out = fs.step(*(t(z["sample"][0][j]) for j in range(3)),
                  model_masks=[t(z["mask_model"][j]) for j in range(4)], d_masks1=[t(z["mask_d1"][j]) for j in range(4)],
                  d_masks2=[t(z["mask_d2"][j]) for j in range(4)], gumbel_u=t(z["gumbel_u"][0]), alpha=t(z["alpha"][0]).view(-1))
    assert abs(float(out["gp"].cpu()) - 0.3) <= 2e-7 * 0.3
    for k, v in fs.D.t.items():
        assert bool(torch.isfinite(v.cpu().double()).all()), k
    for k in fs.hs.P:
        assert bool(torch.isfinite(P[k].cpu()).all()), k


def test_full_step_from_saturated_state_stays_finite():
    full_step_from_saturated_state("cuda")
