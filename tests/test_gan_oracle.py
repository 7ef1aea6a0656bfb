"""oracle/gan_oracle.py (GAN side + full training step, SURVEY 8f row 2) replayed against the trace recorded from three
steps of the unmodified reference `Trainer.train()` (tests/golden/gan_trace.npz, minted by make_golden_gan.py)."""
import json
import os

import numpy as np
import pytest
import scipy.sparse as sp
import torch

from oracle import gan_oracle as GO
from oracle import mmssl_oracle as O
from tests.golden_util import rel_err

TOL = 2e-5      # same torch CPU ops in the same order; slack only for BLAS blocking / accumulation order
# A bias in front of a training-mode BatchNorm has an exactly zero gradient; what autograd returns is cancellation noise
# (1e-2 against weight gradients of 1e4) that Adam then normalises into a +-lr random walk of a parameter no output depends
# on.  Gradients: absolute tolerance at the scale of the layer; state: not compared.
DEAD_BIAS = {"net.0.bias": "net.0.weight", "net.4.bias": "net.4.weight"}


@pytest.fixture(scope="module")
def replay():
    z = np.load(os.path.join(os.path.dirname(__file__), "golden", "gan_trace.npz"))
    c = json.loads(str(z["cfg"]))
    t = lambda a: torch.from_numpy(np.asarray(a))
    P = {k[3:]: t(z[k]) for k in z.files if k.startswith("G0/")}
    S = {k[3:]: t(z[k]).clone() for k in z.files if k.startswith("D0/")}
    R = sp.csr_matrix((np.ones(len(z["train_rows"]), np.float32), (z["train_rows"], z["train_cols"])), shape=(c["U"], c["I"]))
    cfg = O.HotPathConfig(embed_size=c["d"], n_layers=c["n_layers"], head_num=c["head_num"], id_cat_rate=c["id_cat_rate"],
                          model_cat_rate=c["model_cat_rate"], drop_rate=c["drop_rate"], tau=c["tau"], cl_rate=c["cl_rate"],
                          emb_decay=c["emb_decay"], feat_reg_decay=c["feat_reg_decay"], batch_size=c["B"], lr=c["lr"])
    g = GO.GanConfig(G_drop1=c["G_drop1"], G_drop2=c["G_drop2"], gp_rate=c["gp_rate"], G_rate=c["G_rate"], D_lr=c["D_lr"],
                     log_log_scale=c["log_log_scale"], real_data_tau=c["real_data_tau"], ui_pre_scale=c["ui_pre_scale"],
                     m_topk_rate=c["m_topk_rate"], T=c["T"])
    fs = GO.FullStep(P, S, t(z["image_feats"]), t(z["text_feats"]), R, cfg, g)
    traces = []
    for s in range(c["steps"]):
        users, pos, neg = (z["sample"][s][j] for j in range(3))
        traces.append(fs.step(users, pos, neg, [t(z["mask_model"][4 * s + j]) for j in range(4)],
                              [t(z["mask_d1"][4 * s + j]) for j in range(4)], [t(z["mask_d2"][4 * s + j]) for j in range(4)],
                              t(z["gumbel_u"][s]), t(z["alpha"][s])))
    return z, c, traces


def test_u_sim_and_discriminator_calls(replay):
    z, c, traces = replay
    for s, tr in enumerate(traces):
        for j in range(5):
            assert rel_err(tr["u_sim"][j], torch.from_numpy(z["u_sim"][5 * s + j])) < TOL, (s, j)
        for j in range(4):
            assert rel_err(tr["D_in"][j], torch.from_numpy(z["D_in"][4 * s + j])) < TOL, (s, j)
            assert rel_err(tr["D_out"][j], torch.from_numpy(z["D_out"][4 * s + j])) < TOL, (s, j)


def test_gradient_penalty_and_d_step(replay):
    z, c, traces = replay
    for s, tr in enumerate(traces):
        assert abs(float(tr["gp"]) - float(z["gp"][s])) <= TOL * abs(float(z["gp"][s])), s
        for k in GO.D_PARAMS:
            if k in DEAD_BIAS:
                scale = float(np.abs(z["Dgrad/" + DEAD_BIAS[k]][s]).max())
                assert float(tr["Dgrad"][k].abs().max()) < 1e-5 * scale and float(np.abs(z["Dgrad/" + k][s]).max()) < 1e-5 * scale
            else:
                assert rel_err(tr["Dgrad"][k], torch.from_numpy(z["Dgrad/" + k][s])) < 1e-4, (s, k)
        for k in c["d_state_names"]:
            if k in DEAD_BIAS:
                continue
            want = torch.from_numpy(np.asarray(z["Dstate/" + k][s]))
            if k.endswith("running_mean"):      # carries the dead bias of the Linear in front: bounded by its +-lr walk
                assert float((tr["Dstate"][k] - want).abs().max()) <= 1.01 * c["D_lr"] * (s + 1), (s, k)
            elif want.dtype == torch.int64:
                assert int(tr["Dstate"][k]) == int(want)          # BatchNorm num_batches_tracked: 3 calls before the step
            else:
                assert rel_err(tr["Dstate"][k], want) < 1e-4, (s, k)


def test_g_step_gradients_and_parameters(replay):
    z, c, traces = replay
    for s, tr in enumerate(traces):
        for k, gr in tr["Ggrad"].items():
            assert rel_err(gr, torch.from_numpy(z["Ggrad/" + k][s])) < 1e-4, (s, k)
        for k, p in tr["Gparam"].items():
            assert rel_err(p, torch.from_numpy(z["Gparam/" + k][s])) < 1e-4, (s, k)


def test_modality_graph_rebuilds(replay):
    """Step 1 rebuilds from the (users tiled, ids flattened) pairs of step 0; step 2 rebuilds empty graphs."""
    z, c, traces = replay
    assert "graphs" not in traces[0] and int(z["graph_idx/n"]) == 8
    for s in (1, 2):
        for j, gph in enumerate(traces[s]["graphs"]):
            n = 4 * (s - 1) + j
            gc = gph.coalesce()
            assert tuple(gc.shape) == tuple(int(v) for v in z["graph_shape"][n])
            assert np.array_equal(gc.indices().numpy(), z[f"graph_idx/{n}"])
            np.testing.assert_allclose(gc.values().numpy(), z[f"graph_val/{n}"], rtol=1e-6)
    assert traces[1]["graphs"][0]._nnz() > 0 and traces[2]["graphs"][0]._nnz() == 0


# ------------------------------------------------------------------------------------------ closed forms vs autograd
def _random_d(n_items=96, seed=0):
    g = torch.Generator().manual_seed(seed)
    h1, h2 = n_items // 4, n_items // 8
    S = {"net.0.weight": torch.randn(h1, n_items, generator=g) * (2 / n_items) ** 0.5, "net.0.bias": torch.randn(h1, generator=g) * 0.1,
         "net.2.weight": 1 + 0.2 * torch.randn(h1, generator=g), "net.2.bias": 0.1 * torch.randn(h1, generator=g),
         "net.4.weight": torch.randn(h2, h1, generator=g) * (2 / h1) ** 0.5, "net.4.bias": torch.randn(h2, generator=g) * 0.1,
         "net.6.weight": 1 + 0.2 * torch.randn(h2, generator=g), "net.6.bias": 0.1 * torch.randn(h2, generator=g),
         "net.8.weight": torch.randn(1, h2, generator=g) * (2 / h2) ** 0.5, "net.8.bias": torch.zeros(1)}
    for k, n in (("net.2", h1), ("net.6", h2)):
        S[k + ".running_mean"], S[k + ".running_var"] = torch.zeros(n), torch.ones(n)
        S[k + ".num_batches_tracked"] = torch.tensor(0)
    return {k: v.double() if v.is_floating_point() else v for k, v in S.items()}, g


def test_closed_form_first_order_backward_matches_autograd():
    S, g = _random_d()
    n, I = 48, 96
    x = torch.randn(n, I, generator=g).double()
    m1 = ((torch.rand(n, I // 4, generator=g) >= 0.31) / 0.69).double()
    m2 = ((torch.rand(n, I // 8, generator=g) >= 0.5) / 0.5).double()
    dout = torch.randn(n, generator=g).double()
    Sa = {k: (v.clone().requires_grad_(True) if k in GO.D_PARAMS else v.clone()) for k, v in S.items()}
    xa = x.clone().requires_grad_(True)
    out = GO.discriminator(xa, Sa, m1, m2)
    want = torch.autograd.grad((out * dout).sum(), [Sa[k] for k in GO.D_PARAMS] + [xa])
    c = GO.d_forward_cache(x, S, m1, m2)
    assert rel_err(c["out"], out) < 1e-12
    got, dx, _ = GO.d_backward(c, S, dout, need_dx=True)
    for k, w in zip(GO.D_PARAMS, want):
        if k in DEAD_BIAS:
            assert float(got[k].abs().max()) < 1e-9 and float(w.abs().max()) < 1e-9
        else:
            assert rel_err(got[k].view_as(w), w) < 1e-10, k
    assert rel_err(dx, want[-1]) < 1e-10


def test_closed_form_gradient_penalty_matches_double_backward():
    """Explicit reverse sweep over [forward ; backward] (BatchNorm statistics included) == autograd's double backward."""
    S, g = _random_d(seed=4)
    n, I = 64, 96
    xr = torch.nn.functional.normalize(torch.rand(n, I, generator=g).double(), dim=1)
    xf = torch.nn.functional.normalize(torch.randn(n, I, generator=g).double(), dim=1)
    alpha = torch.rand(n, 1, generator=g).double()
    m1 = ((torch.rand(n, I // 4, generator=g) >= 0.31) / 0.69).double()
    m2 = ((torch.rand(n, I // 8, generator=g) >= 0.5) / 0.5).double()
    Sa = {k: (v.clone().requires_grad_(True) if k in GO.D_PARAMS else v.clone()) for k, v in S.items()}
    gp_a = GO.gradient_penalty(Sa, xr, xf, alpha, m1, m2, GO.GanConfig())
    want = torch.autograd.grad(gp_a, [Sa[k] for k in GO.D_PARAMS], allow_unused=True)
    inter = alpha * xr + (1 - alpha) * xf
    gp_c, G = GO.gradient_penalty_closed(inter, S, m1, m2, lam=0.3)
    assert abs(float(gp_c) - float(gp_a)) < 1e-12 * max(1.0, abs(float(gp_a)))
    scale = max(float(w.abs().max()) for w in want if w is not None)
    for k, w in zip(GO.D_PARAMS, want):
        if w is None:                                  # the last bias does not reach d out / d x
            assert float(G[k].abs().max()) == 0.0, k
        elif k in DEAD_BIAS:
            assert float(G[k].abs().max()) < 1e-9 * scale
        else:
            assert rel_err(G[k].view_as(w), w) < 1e-9, k


def test_closed_form_gradient_penalty_with_saturated_heads():
    """Every head saturated (sigmoid == 1 exactly): d out / d x is exactly zero on every row.  Autograd's norm backward gives
    such a row a zero gradient, so gp = lambda and every penalty gradient is 0; the closed form must not turn (-inf) * 0
    into NaN."""
    S, g = _random_d(seed=5)
    S["net.8.bias"] = torch.full((1,), 60.0, dtype=torch.float64)      # sigmoid(z) == 1 in float64 for z > 37
    n, I = 32, 96
    xr = torch.nn.functional.normalize(torch.rand(n, I, generator=g).double(), dim=1)
    xf = torch.nn.functional.normalize(torch.randn(n, I, generator=g).double(), dim=1)
    alpha = torch.rand(n, 1, generator=g).double()
    m1 = ((torch.rand(n, I // 4, generator=g) >= 0.31) / 0.69).double()
    m2 = ((torch.rand(n, I // 8, generator=g) >= 0.5) / 0.5).double()
    Sa = {k: (v.clone().requires_grad_(True) if k in GO.D_PARAMS else v.clone()) for k, v in S.items()}
    gp_a = GO.gradient_penalty(Sa, xr, xf, alpha, m1, m2, GO.GanConfig())
    want = torch.autograd.grad(gp_a, [Sa[k] for k in GO.D_PARAMS], allow_unused=True)
    assert float(gp_a) == 0.3 and all(w is None or float(w.abs().max()) == 0.0 for w in want)
    gp_c, G = GO.gradient_penalty_closed(alpha * xr + (1 - alpha) * xf, S, m1, m2, lam=0.3)
    assert float(gp_c) == 0.3
    for k in GO.D_PARAMS:
        assert bool(torch.isfinite(G[k]).all()) and float(G[k].abs().max()) == 0.0, k


def test_gp_rows_spec_on_zero_and_unit_rows_matches_autograd():
    """tests/gan_ops_cpu.gp_rows (the kernel's specification) against autograd of lam * mean((||g|| - 1)^2) in float64, on
    rows of norm 0, rows of norm exactly 1 and rows of 1e-20 next to ordinary rows."""
    from tests import gan_ops_cpu as REF
    g = torch.Generator().manual_seed(8)
    n, w = 10, 7
    gx = torch.randn(n, w, generator=g, dtype=torch.float64)
    gx[1] = 0.0
    gx[4] = 0.0
    gx[2] = 0.0
    gx[2, 3] = 1.0                                     # norm exactly 1: zero gradient, zero penalty
    gx[6] = 1e-20 * torch.randn(w, generator=g, dtype=torch.float64)
    ga = gx.clone().requires_grad_(True)
    gp_a = 0.3 * ((ga.norm(2, dim=1) - 1) ** 2).mean()
    want = torch.autograd.grad(gp_a, ga)[0]
    gp, gbar = REF.gp_rows(gx, 0.3)
    assert abs(float(gp) - float(gp_a)) < 1e-15 and bool(torch.isfinite(gbar).all())
    assert float(gbar[1].abs().max()) == 0.0 and float(gbar[4].abs().max()) == 0.0 and float(gbar[2].abs().max()) == 0.0
    assert rel_err(gbar, want) < 1e-14


def test_float64_full_step_runs_in_float64():
    """FullStep(dtype=torch.float64) casts state, features, graphs and draws: every recorded result is float64, and one
    iteration agrees with the fp32 oracle to fp32 accuracy."""
    from tests import fullstep_check
    z, c = fullstep_check.load_trace()
    t = lambda a: torch.from_numpy(np.asarray(a)).clone()
    R = sp.csr_matrix((np.ones(len(z["train_rows"]), np.float32), (z["train_rows"], z["train_cols"])), shape=(c["U"], c["I"]))
    cfg = O.HotPathConfig(embed_size=c["d"], n_layers=c["n_layers"], head_num=c["head_num"], id_cat_rate=c["id_cat_rate"],
                          model_cat_rate=c["model_cat_rate"], drop_rate=c["drop_rate"], tau=c["tau"], cl_rate=c["cl_rate"],
                          emb_decay=c["emb_decay"], feat_reg_decay=c["feat_reg_decay"], batch_size=c["B"], lr=c["lr"])
    g = GO.GanConfig(G_rate=c["G_rate"], D_lr=c["D_lr"], gp_rate=c["gp_rate"], m_topk_rate=c["m_topk_rate"], T=c["T"])
    P = {k[3:]: t(z[k]) for k in z.files if k.startswith("G0/")}
    S = {k[3:]: t(z[k]) for k in z.files if k.startswith("D0/")}
    runs = {}
    for dt in (torch.float32, torch.float64):
        fs = GO.FullStep(P, S, t(z["image_feats"]), t(z["text_feats"]), R, cfg, g, dtype=dt)
        users, pos, neg = (z["sample"][0][j] for j in range(3))
        runs[dt] = fs.step(users, pos, neg, [t(z["mask_model"][j]) for j in range(4)], [t(z["mask_d1"][j]) for j in range(4)],
                           [t(z["mask_d2"][j]) for j in range(4)], t(z["gumbel_u"][0]), t(z["alpha"][0]))
    lo, hi = runs[torch.float32], runs[torch.float64]
    assert hi["gp"].dtype == torch.float64 and all(v.dtype == torch.float64 for v in hi["Ggrad"].values())
    assert all(x.dtype == torch.float64 for x in hi["u_sim"] + hi["D_out"])
    assert abs(float(lo["gp"]) - float(hi["gp"])) < 1e-4 * abs(float(hi["gp"]))
    for k in GO.D_PARAMS:
        if k not in DEAD_BIAS:
            assert rel_err(lo["Dgrad"][k], hi["Dgrad"][k]) < 1e-4, k
    for k in hi["Ggrad"]:
        assert rel_err(lo["Ggrad"][k], hi["Ggrad"][k]) < 1e-4, k


def test_d_step_grads_matches_full_step_trace(replay):
    """gan_oracle.d_step_grads (the yardstick of the device's composite D step) == the D gradients FullStep records."""
    z, c, traces = replay
    S = {k[3:]: torch.from_numpy(np.asarray(z[k])).clone() for k in z.files if k.startswith("D0/")}
    B = c["B"]
    tr = traces[0]
    t = lambda a: torch.from_numpy(np.asarray(a))
    res = GO.d_step_grads(S, tr["D_in"][0], tr["D_in"][1], t(z["alpha"][0]), [t(z["mask_d1"][j]) for j in range(3)],
                          [t(z["mask_d2"][j]) for j in range(3)], GO.GanConfig(gp_rate=c["gp_rate"]))
    assert abs(float(res["gp"]) - float(tr["gp"])) <= 1e-6 * abs(float(tr["gp"]))
    for j in range(3):
        assert rel_err(res["outs"][j], tr["D_out"][j]) < 1e-6
    for k in GO.D_PARAMS:
        if k not in DEAD_BIAS:
            assert rel_err(res["grads"][k], tr["Dgrad"][k]) < 1e-6, k
    assert tr["D_in"][1].shape[0] == 2 * B


def test_closed_form_u_sim_backward_matches_autograd():
    g = torch.Generator().manual_seed(2)
    U, I, d, B = 40, 50, 16, 12
    R = sp.random(U, I, density=0.1, format="csr", random_state=1, dtype=np.float32)
    R.data[:] = 1.0
    uf = torch.randn(U, d, generator=g, dtype=torch.float64, requires_grad=True)
    itf = torch.randn(I, d, generator=g, dtype=torch.float64, requires_grad=True)
    users = torch.randperm(U, generator=g)[:B].tolist()
    go = torch.randn(B, I, generator=g, dtype=torch.float64)
    R64 = R.astype(np.float64)
    out = GO.u_sim(users, uf, itf, R64, batch_size=16)
    wu, wi = torch.autograd.grad((out * go).sum(), [uf, itf])
    du_rows, di = GO.u_sim_backward(users, uf.detach(), itf.detach(), R64, go)
    assert rel_err(du_rows, wu[users]) < 1e-10 and rel_err(di, wi) < 1e-10
