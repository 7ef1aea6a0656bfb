"""The training hot step (mmssl_b200/hotstep.py: forward, BPR + 2 x InfoNCE + feat_reg, hand-written backward, AdamW) against
float64, with the yardstick of tests/hotstep_fp64.py: a device result may be 4x as far from float64 as fp32 autograd of the
oracle on the same inputs, with a floor per route, norm-wise, row-wise and per class of rows.

  a. each loss term alone or dominant (a term worth 1e-5 of the gradient is invisible at 1e-4 of the largest entry);
  b. a shape where every class of rows is populated, every width, K, head count, modality-graph state and route;
  c. legitimate but awkward batches (repeated users, pos == neg, an item both positive and negative, rows without an edge,
     batch sizes across the InfoNCE route boundary, evaluation mode, no dropout, saturated scores);
  d. replays with a new batch and new masks each time, every one checked from the device's own parameters;
  e. the AdamW update from the device's own gradient: moments and displacement against a float64 AdamW.

The check_* bodies also run on the CPU under the cuemu emulator at small sizes (tests/test_emu_hotstep_fp64.py)."""
import math
from dataclasses import replace

import numpy as np
import pytest
import torch

from tests import hotstep_fp64 as H

pytestmark = pytest.mark.gpu
ROUTES = ("simt/simt", "simt/auto", "tc/simt", "tc/auto")
WIDTHS = (32, 64, 96, 128, 192, 256)
MODALS = ("alias", "distinct", "empty")


def _cfg(d=64, K=2, B=96, **kw):
    from mmssl_b200.hotstep import HotStepConfig
    return HotStepConfig(embed_size=d, n_layers=K, batch_size=B, **kw)


def routes_for(d):
    """Tensor-core InfoNCE exists at d = 64 and 128 only: elsewhere 'auto' is the CUDA-core route again."""
    return ROUTES if d in (64, 128) else ("simt/simt", "tc/simt")


# ------------------------------------------------------------------------------------------------ a. term isolation
def term_configs(I, B):
    return {
        "default": {},
        "bpr only": dict(cl_rate=0.0, emb_decay=0.0, feat_reg_decay=0.0),
        "emb_reg dominant": dict(emb_decay=1e2),
        "feat_reg dominant": dict(feat_reg_decay=float(I)),
        "infonce dominant": dict(cl_rate=1e2),
        "id_cat_rate 0": dict(id_cat_rate=0.0),
        "model_cat_rate 0": dict(model_cat_rate=0.0),
        "configured batch_size != batch": dict(batch_size=7 * B + 1),     # the regulariser divides by the configured size
        "tau 0.2": dict(tau=0.2),
    }


TERMS = tuple(term_configs(1, 1))


def check_terms(term, route, modal="distinct", U=523, I=391, B=96, d=64, cuts=H.DEFAULT_CUTS):
    p = H.problem(U, I, d=d, B=B, modal=modal, seed=11, cuts=cuts)
    cfg = replace(_cfg(d, 2, B), **term_configs(I, B)[term])
    hs = H.hot_step(p, cfg, route)
    hi, _ = H.check_step(hs, p, cfg, route, what=f"{term} {modal}")
    if term == "emb_reg dominant":          # the configuration does what it is for
        assert float(hi["losses"][2]) > 10 * float(hi["losses"][1])
    if term == "bpr only":
        assert float(hs.out5[2]) == 0.0 and float(hs.out5[3]) == 0.0


@pytest.mark.parametrize("route", ROUTES)
@pytest.mark.parametrize("term", TERMS)
def test_each_loss_term(term, route):
    check_terms(term, route)


# ------------------------------------------------------------------------------------------------ b. row classes
def check_row_classes(d, K, head_num, modal, route, U=1531, I=1237, B=257, dv=72, dt=40, cuts=H.DEFAULT_CUTS, set_cuts=None):
    if set_cuts is not None:
        set_cuts(*cuts)
    assert U % 4 and I % 4 and dv % 64 and dt % 64
    p = H.problem(U, I, d=d, B=B, modal=modal, dv=dv, dt=dt, head_num=head_num, seed=d + K, cuts=cuts)
    cls = H.row_classes(p)
    for table in (H.P_EU, H.P_EI):          # every class has rows, in both tables
        for name, m in cls[table].items():
            assert int(m.sum()) > 0, (table, name)
    cfg = _cfg(d, K, B, head_num=head_num)
    hs = H.hot_step(p, cfg, route)
    g = hs.graphs[0]
    assert g.fwd.n_split_rows >= 4 and g.bwd.n_split_rows >= 4       # the plan did split them, in both directions
    H.check_step(hs, p, cfg, route, what=f"d={d} K={K} H={head_num} {modal}", outs=True)


def row_class_cases():
    out = []
    for j, d in enumerate(WIDTHS):
        for m, modal in enumerate(MODALS):
            K, heads = 1 + (j + m) % 4, (1, 4)[(j + m) % 2]
            out += [(d, K, heads, modal, r) for r in routes_for(d)]
    return out


@pytest.mark.parametrize("d,K,head_num,modal,route", row_class_cases())
def test_row_classes(d, K, head_num, modal, route):
    check_row_classes(d, K, head_num, modal, route)


@pytest.mark.parametrize("name", ["baby", "sports"])
def test_full_size_distinct_graphs(name):
    """One step at the Baby / Sports shape with distinct modality graphs; rows by class, from the data set's own degrees."""
    from mmssl_b200.synthetic import CONFIGS, make_bipartite
    torch.set_num_threads(8)
    U, I, nnz, d, K, dv, dt = CONFIGS[name]
    p = H.problem(U, I, d=d, B=1024, modal="distinct", dv=dv, dt=dt, seed=2022, train=make_bipartite(U, I, nnz, seed=2022))
    cfg = _cfg(d, K, 1024)
    for route in ("tc/auto", "simt/simt"):
        hs = H.hot_step(p, cfg, route)
        H.check_step(hs, p, cfg, route, what=f"{name}")
        del hs


# ------------------------------------------------------------------------------------------------ c. awkward batches
AWKWARD = ("repeated users", "pos == neg", "positive and negative", "no edge", "evaluation", "no dropout", "saturated")


def check_awkward(kind, route, U=523, I=391, B=96, d=64, modal="alias", cuts=H.DEFAULT_CUTS):
    p = H.problem(U, I, d=d, B=B, modal=modal, seed=5, cuts=cuts, table_scale=30.0 if kind == "saturated" else 1.0)
    u, po, ne = p.users.clone(), p.pos.clone(), p.neg.clone()
    cfg, training = _cfg(d, 2, B), True
    if kind == "repeated users":            # what the sampler draws when B > users with an item: identical InfoNCE rows
        u[B // 2:] = u[:B - B // 2]
        u[1] = u[0]
    elif kind == "pos == neg":
        ne[::3] = po[::3]
    elif kind == "positive and negative":   # g_p and g_n are one buffer
        ne[1:] = po[:-1]
    elif kind == "no edge":                 # zero rows: F.normalize's eps clamp, the 1/d softmax row
        u[0], po[1], ne[2] = U - 2, I - 2, I - 2
    elif kind == "evaluation":
        training = False
    elif kind == "no dropout":
        cfg = replace(cfg, drop_rate=0.0)
    p = p.with_batch(u, po, ne)
    hs = H.hot_step(p, cfg, route, training=training)
    hi, _ = H.check_step(hs, p, cfg, route, what=kind)
    if kind == "saturated":                 # the state does what it is for: some BPR sigmoids are saturated in fp32
        s = (hi["outs"][0][p.users] * (hi["outs"][1][p.pos] - hi["outs"][1][p.neg])).sum(1)
        assert float(s.abs().max()) > 17.0, float(s.abs().max())


@pytest.mark.parametrize("route", ROUTES)
@pytest.mark.parametrize("kind", AWKWARD)
def test_awkward_batches(kind, route):
    check_awkward(kind, route)


def check_batch_size(B, route, U=1531, I=1237, d=64, cuts=H.DEFAULT_CUTS):
    p = H.problem(U, I, d=d, B=B, modal="alias", seed=B, cuts=cuts)
    cfg = _cfg(d, 2, B)
    hs = H.hot_step(p, cfg, route)
    assert hs.nce[0].tc == (route.endswith("auto") and B <= 2048)
    if B > 1:
        return H.check_step(hs, p, cfg, route, what=f"B={B}")
    # B = 1: the InfoNCE value is -1e-8 and its gradient 0 exactly; what the device leaves is the cancellation residue of
    # e^(1/tau) that tests/test_gpu_zz_route_parity.py bounds by 2^-16 e^(1/tau).  Value absolutely; gradients by the rule.
    hi, lo = H.both(p, cfg)
    out5 = hs.run().double().cpu()
    resid = 2.0 ** -16 * math.exp(1.0 / cfg.tau)
    assert abs(float(out5[4]) - float(hi["losses"][4])) < resid
    for j in (1, 2, 3):
        assert abs(float(out5[j]) - float(hi["losses"][j])) <= 1e-5 * abs(float(hi["losses"][j]))
    cls = H.row_classes(p)
    floor = dict(H.FLOOR[route])
    # the residue lands on rows whose own gradient is small: row-wise 4x the route's floor (measured 1.0e-4, text_trans.weight, tc)
    H.FLOOR[route] = dict(floor, norm=max(floor["norm"], cfg.cl_rate * resid), row=4 * floor["row"])
    try:
        for k in H.LIVE:
            H.assert_close(k + " (B=1)", hs.grads[k], lo["grads"][k], hi["grads"][k], route, cls.get(k), "B=1")
    finally:
        H.FLOOR[route] = floor


@pytest.mark.parametrize("route", ["simt/simt", "tc/auto"])
@pytest.mark.parametrize("B", [1, 2, 63, 65, 257, 1000, 1024, 1025, 2048, 2049])
def test_batch_sizes(B, route):
    check_batch_size(B, route)


# ------------------------------------------------------------------------------------------------ d. replays
def check_replays(modal, route, mode, U=523, I=391, B=96, d=64, n=8, cuts=H.DEFAULT_CUTS):
    """`n` optimiser steps, each with another batch and other masks, each compared with float64 evaluated at the parameters
    the device held before that step.  mode: 'eager', 'graph' (one capture, n replays; an eager twin must give the same
    losses) or 'sampler' (captured, batches drawn on the device)."""
    from mmssl_b200.synthetic import TripleSampler
    p = H.problem(U, I, d=d, B=B, modal=modal, seed=3, cuts=cuts)
    cfg = _cfg(d, 2, B)
    smp = None
    if mode == "sampler":
        from mmssl_b200.sampler import DeviceTripleSampler
        smp = DeviceTripleSampler(p.train, seed=17)
    graphs = H.device_graphs(p)
    hs = H.hot_step(p, cfg, route, optimizer_step=True, sampler=smp, graphs=graphs)
    twin = H.hot_step(p, cfg, route, optimizer_step=True, graphs=graphs) if mode == "graph" else None
    assert hs.engine is not None and (modal != "empty" or not any(g.nnz for g in hs.graphs[2:]))
    if mode != "eager":
        hs.capture(warmup=1)                # the warm-up step is an optimiser step too
        if twin is not None:
            twin.run()
    draw = TripleSampler(p.train, seed=29)
    gen = torch.Generator().manual_seed(41)
    for r in range(n):
        masks = H.new_masks(I, d, cfg.drop_rate, gen)
        batch = draw.sample(B)
        if r == n - 1:                      # the last one repeats users and shares items between the roles
            batch[0][B // 2:] = batch[0][:B - B // 2]
            batch[2][1:] = batch[1][:-1]
        for dst, src in zip(hs.masks, masks):
            dst.copy_(src)
        hs.set_indices(*batch)
        before = {k: v.detach().cpu().clone() for k, v in hs.P.items()}
        out5 = (hs.run() if mode == "eager" else hs.replay()).clone()
        torch.cuda.synchronize()
        if smp is not None:
            batch = tuple(t.cpu().numpy() for t in hs.idx)
        q = p.with_batch(*batch, masks=masks)
        H.check_step(hs, q, cfg, route, what=f"{mode} replay {r} {modal}", out5=out5, params=before)
        assert int(hs.step_dev.cpu()[0]) == r + (1 if mode == "eager" else 2)
        if twin is not None:
            for dst, src in zip(twin.masks, masks):
                dst.copy_(src)
            twin.set_indices(*batch)
            e5 = twin.run().double().cpu()
            err = float(((e5 - out5.double().cpu()).abs() / e5.abs().clamp_min(1e-30)).max())
            assert err < 1e-5, (r, err, e5.tolist(), out5.tolist())       # same arithmetic, atomics in another order


@pytest.mark.parametrize("route", ["tc/auto", "simt/simt"])
@pytest.mark.parametrize("mode", ["eager", "graph", "sampler"])
@pytest.mark.parametrize("modal", ["distinct", "empty", "alias"])
def test_replays_from_device_state(modal, mode, route):
    check_replays(modal, route, mode)


# ------------------------------------------------------------------------------------------------ e. AdamW
def _adamw_refs(p0, g, m0, v0, step, lr, b1, b2, eps, wd):
    """(P, m, v) after one update in float64 (the oracle's adamw_step) and by torch.optim.AdamW in fp32 from the same state.
    Both take the betas the kernel receives: the C ABI carries them as fp32, and 1 - float(0.999) is 1.3e-5 from 0.001, so an
    AdamW with the decimal beta2 has a second moment 1.3e-5 from the kernel's (a hyper-parameter moved by 1.3e-8, not an error
    of the arithmetic)."""
    b1, b2 = float(np.float32(b1)), float(np.float32(b2))
    p64, m64, v64 = p0.double().clone(), m0.double().clone(), v0.double().clone()
    H.O.adamw_step(p64, g.double(), m64, v64, step, lr, wd, b1, b2, eps)
    p32 = p0.clone().requires_grad_(True)
    opt = torch.optim.AdamW([p32], lr=lr, betas=(b1, b2), eps=eps, weight_decay=wd, foreach=False)
    opt.state[p32] = dict(step=torch.tensor(float(step - 1)), exp_avg=m0.clone(), exp_avg_sq=v0.clone())
    p32.grad = g.clone()
    opt.step()
    st = opt.state[p32]
    return (p64, m64, v64), (p32.detach(), st["exp_avg"], st["exp_avg_sq"])


def assert_update(name, p0, got, hi, lo):
    """Moments norm-wise by the 4x rule (floor 2^-22); the displacement P_after - P_before, whose fp32 storage carries half an
    ulp of P, within that half ulp plus 4x what torch's fp32 AdamW shows."""
    p0 = p0.double()
    for j, what in ((1, "m"), (2, "v")):
        scale = max(float(hi[j].abs().max()), 1e-300)
        e, ref = float((got[j].double() - hi[j]).abs().max()) / scale, float((lo[j].double() - hi[j]).abs().max()) / scale
        assert e <= max(H.K_FP32 * ref, 2.0 ** -22), f"{name} {what}: device {e:.3g}, torch fp32 {ref:.3g}"
    disp, d64, d32 = got[0].double() - p0, hi[0] - p0, lo[0].double() - p0
    half_ulp = torch.maximum(got[0].abs(), p0.float().abs()).double() * 2.0 ** -24 + 1e-45
    e = float(((disp - d64).abs() - half_ulp).max())
    ref = float((d32 - d64).abs().max())
    assert e <= H.K_FP32 * ref, (f"{name} displacement: device {float((disp - d64).abs().max()):.3g} from float64, "
                                f"torch fp32 {ref:.3g}, largest displacement {float(d64.abs().max()):.3g}")
    return float((disp - d64).abs().max()), ref


def check_adamw_in_step(step, wd, lr, route="simt/simt", U=203, I=157, B=48, d=64):
    """One HotStep with the optimiser, resumed at `step` - 1 with non-trivial moments: the update from the device's own
    gradient (hs.grads is what the kernel read) against float64."""
    p = H.problem(U, I, d=d, B=B, modal="distinct", seed=step % 97)
    cfg = replace(_cfg(d, 2, B), weight_decay=wd, lr=lr)
    hs = H.hot_step(p, cfg, route, optimizer_step=True)
    gen = torch.Generator().manual_seed(step)
    state = hs.state_dict()
    cpu = lambda dct: {k: v.detach().cpu().clone() for k, v in dct.items()}
    optim = dict(m=cpu(state["optim"]["m"]), v=cpu(state["optim"]["v"]), step=step - 1)
    if step > 1:                            # moments of the size a run leaves: |m| ~ 1e-3 sqrt(v) .. sqrt(v)
        for k in H.LIVE:
            optim["v"][k] = (torch.rand(optim["v"][k].shape, generator=gen) * 1e-6 + 1e-12)
            optim["m"][k] = torch.randn(optim["m"][k].shape, generator=gen) * optim["v"][k].sqrt()
    hs.load_state_dict(dict(state, model=cpu(state["model"]), optim=optim))
    p0 = cpu(hs.P)
    hs.run()
    assert int(hs.step_dev.cpu()[0]) == step
    worst = {}
    for k in H.LIVE:
        g = hs.grads[k].cpu()
        hi, lo = _adamw_refs(p0[k], g, optim["m"][k], optim["v"][k], step, lr, cfg.beta1, cfg.beta2, cfg.eps, wd)
        worst[k] = assert_update(f"step {step} wd {wd} lr {lr} {k}", p0[k], (hs.P[k].cpu(), hs.m[k].cpu(), hs.v[k].cpu()), hi, lo)
    return worst


@pytest.mark.parametrize("lr", [5.5e-4, 1e-1])
@pytest.mark.parametrize("wd", [0.0, 1e-2, 1.0])
@pytest.mark.parametrize("step", [1, 2, 10, 1000, 100000])
def test_adamw_update_in_step(step, wd, lr):
    check_adamw_in_step(step, wd, lr)


def check_adamw_many_tensors(gan=False):
    """19 tensors in one ops.adamw call (the wrapper sends 16 + 3), sizes with numel % 4 in {1, 2, 3} on both sides of the
    boundary; through gan_ops.adam with the Discriminator's hyper-parameters when `gan`."""
    from mmssl_b200 import gan as G, gan_ops, ops
    gen = torch.Generator().manual_seed(7)
    sizes = [8, 1, 64, 5, 1027, 12, 3, 256, 2, 33, 4, 7, 130, 6, 9, 1001, 1002, 1003, 11]
    assert len(sizes) > 16 and {sizes[j] % 4 for j in (14, 15, 16, 17)} == {1, 2, 3}
    p0 = [torch.randn(n, generator=gen) for n in sizes]
    g = [torch.randn(n, generator=gen) * 1e-2 for n in sizes]
    m0 = [torch.randn(n, generator=gen) * 1e-3 for n in sizes]
    v0 = [torch.rand(n, generator=gen) * 1e-5 for n in sizes]
    dev = lambda ts: [t.clone().cuda() for t in ts]
    P, Gd, M, V = dev(p0), dev(g), dev(m0), dev(v0)
    step = 5
    if gan:
        hp = G.GanHyper()
        lr, b1, b2, eps, wd = hp.D_lr, hp.beta1, hp.beta2, 1e-8, 0.0
        gan_ops.adam(P, Gd, M, V, step, lr, b1, b2)
    else:
        lr, b1, b2, eps, wd = 5.5e-4, 0.9, 0.999, 1e-8, 1e-2
        ops.adamw(P, Gd, M, V, torch.full((1,), step, dtype=torch.int32).cuda(), lr, b1, b2, eps, wd)
    for j, n in enumerate(sizes):
        hi, lo = _adamw_refs(p0[j], g[j], m0[j], v0[j], step, lr, b1, b2, eps, wd)
        assert_update(f"tensor {j} numel {n}", p0[j], (P[j].cpu(), M[j].cpu(), V[j].cpu()), hi, lo)


@pytest.mark.parametrize("gan", [False, True])
def test_adamw_many_tensors(gan):
    check_adamw_many_tensors(gan)


def check_adamw_zero_gradient():
    """Zero gradient, zero moments: the update is the decay alone, P * (1 - lr * wd) rounded once, and the moments stay 0."""
    from mmssl_b200 import ops
    gen = torch.Generator().manual_seed(9)
    for lr, wd in ((5.5e-4, 1e-2), (1e-1, 1.0), (5.5e-4, 0.0)):
        p0 = torch.randn(1003, generator=gen)
        P, Z, M, V = p0.clone().cuda(), torch.zeros(1003).cuda(), torch.zeros(1003).cuda(), torch.zeros(1003).cuda()
        ops.adamw([P], [Z], [M], [V], torch.full((1,), 3, dtype=torch.int32).cuda(), lr, 0.9, 0.999, 1e-8, wd)
        decay = np.float32(1.0) - np.float32(lr) * np.float32(wd)
        assert np.array_equal(P.cpu().numpy(), p0.numpy() * decay), (lr, wd)
        assert float(M.abs().max()) == 0.0 and float(V.abs().max()) == 0.0


def test_adamw_zero_gradient_is_exactly_the_decay():
    check_adamw_zero_gradient()


def test_zz_report_distances():
    """Largest distances to float64 seen by this module's tests, per route, tensor and measure (shown with -s)."""
    print("\n" + H.report())
