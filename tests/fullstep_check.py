"""Shared body of the full-step parity tests (GPU: tests/test_gpu_zz_fullstep.py, CPU emulation: tests/test_emu_fullstep.py):
``mmssl_b200.fullstep.FullStep`` replayed against the 3-iteration trace recorded from the UNMODIFIED reference trainer
(tests/golden/gan_trace.npz, minted by tests/golden/make_gan_trace.py) with every random draw injected."""
import json
import os

import numpy as np
import scipy.sparse as sp
import torch

from tests.golden_util import rel_err

TOL = 1e-4                                            # north_star: 1e-4 relative fp32
DEAD_BIAS = {"net.0.bias": "net.0.weight", "net.4.bias": "net.4.weight"}     # exactly-zero gradients (bias before BatchNorm)
# Lowest bound of a GAN-side result against float64, per GEMM route.  All-fp32 routes: 2e-5 (a bias gradient of the D step
# is a column sum with cancellation; measured on the H100: net.6.bias 1.2e-5 at I = 16, B = 24, fp32 autograd 1.8e-6).  The
# tensor-core route carries 2^-17 per bf16 hi/lo operand and 4.7e-6 to 1.4e-5 per product from its accumulation passes
# (DESIGN section 4), and the D gradients are cancelling sums of several such products: measured up to 5.6e-4 (net.8.bias,
# fp32 autograd 1.6e-5), so 1e-3 there.  Both are the numbers DESIGN section 2 reports.
FP64_FLOOR = {"simt": 2e-5, "cublas": 2e-5, "tc": 1e-3}


def within_fp32_reach(got, want64, ref32, floor, what, scale=None):
    """``got`` (device) against the float64 value ``want64``, bounded by what fp32 achieves on the same problem: at most 4x the
    distance of ``ref32`` (the fp32 autograd oracle on the same inputs) to float64, never below ``floor``.  Returns both
    distances: max-norm relative (``rel_err``), or max |difference| / ``scale`` when a scale is given."""
    if scale is None:
        e_dev, e_32 = rel_err(got, want64), rel_err(ref32, want64)
    else:
        d = lambda a: float((a.detach().double().cpu() - want64.double()).abs().max()) / scale
        e_dev, e_32 = d(got), d(ref32)
    bound = max(4.0 * e_32, floor)
    assert e_dev <= bound, f"{what}: device {e_dev:.3g} vs float64, fp32 oracle {e_32:.3g} vs float64, bound {bound:.3g}"
    return e_dev, e_32


def d_step_vs_float64(S, dres, ui, img, txt, users, R, gu, al, m1, m2, gcfg, floor, what=""):
    """One device D step (``dres``: gp, lossf_sum, lossr_sum, grads -- from gan.d_step or FullStep) against the float64
    autograd of the reference's D step on the same state ``S`` (taken before the step), the same u_sim rows (the device's
    own, so that only the D step is measured) and the same masks, Gumbel draws and alpha.  The fp32 autograd oracle on the
    same inputs sets the bound (``within_fp32_reach``).  Returns {name: (device distance, fp32 oracle distance)}."""
    from oracle import gan_oracle as GO
    cpu = lambda x: x.detach().cpu()
    users = [int(u) for u in cpu(users)]
    ui, img, txt, gu, al = (cpu(x) for x in (ui, img, txt, gu, al))
    m1, m2 = [cpu(m) for m in m1[:3]], [cpu(m) for m in m2[:3]]
    res = {}
    for dt in (torch.float64, torch.float32):
        Sd = {k: (cpu(v).to(dt) if v.is_floating_point() else cpu(v)) for k, v in S.items()}
        rr = GO.real_rows(users, R, gu.to(dt), ui.to(dt), gcfg)
        res[dt] = GO.d_step_grads(Sd, torch.cat((img, txt)).to(dt), torch.cat((rr, rr)), al.to(dt), m1, m2, gcfg)
    hi, lo = res[torch.float64], res[torch.float32]
    n = img.shape[0] * 2
    dist = {"gp": within_fp32_reach(cpu(dres["gp"]).view(1), hi["gp"].view(1), lo["gp"].view(1), floor, f"{what} gp")}
    for j, key in ((0, "lossf_sum"), (1, "lossr_sum")):
        if key not in dres:
            continue
        dist[key] = within_fp32_reach(cpu(dres[key]).view(1) * 100.0, hi["outs"][j].sum().view(1), lo["outs"][j].sum().view(1),
                                      floor, f"{what} {key}")
    for k in GO.D_PARAMS:
        got = cpu(dres["grads"][k]).view_as(hi["grads"][k])
        if k in DEAD_BIAS:       # exactly zero in exact arithmetic: cancellation noise, at most 4x the fp32 oracle's own
            scale = float(hi["grads"][DEAD_BIAS[k]].abs().max())
            noise, noise32 = float(got.abs().max()), float(lo["grads"][k].abs().max())
            assert bool(torch.isfinite(got).all()) and noise <= max(4 * noise32, floor * scale), (what, k, noise, noise32, scale)
        elif k.endswith(".bias"):
            # a bias gradient is a row sum of the terms its layer's weight gradient sums against the inputs, often cancelling
            # to a small value (net.8.bias is one such sum): measured at the scale of the layer
            scale = max(float(hi["grads"][k].abs().max()), float(hi["grads"][k[:-4] + "weight"].abs().max()), 1e-30)
            dist[k] = within_fp32_reach(got, hi["grads"][k], lo["grads"][k], floor, f"{what} {k}", scale=scale)
        else:
            dist[k] = within_fp32_reach(got, hi["grads"][k], lo["grads"][k], floor, f"{what} {k}")
    assert n == hi["outs"][0].numel()
    return dist


def load_trace():
    z = np.load(os.path.join(os.path.dirname(__file__), "golden", "gan_trace.npz"))
    return z, json.loads(str(z["cfg"]))


def build(z, c, dev, proj_impl="tc"):
    from mmssl_b200 import gan
    from mmssl_b200.engine import FeatureStore
    from mmssl_b200.fullstep import FullStep, FullStepConfig
    from mmssl_b200.graph import BipartiteGraph
    from mmssl_b200.hotstep import HotStepConfig
    from mmssl_b200.synthetic import csr_norm
    t = lambda a: torch.from_numpy(np.asarray(a)).clone().to(dev)
    R = sp.csr_matrix((np.ones(len(z["train_rows"]), np.float32), (z["train_rows"], z["train_cols"])), shape=(c["U"], c["I"]))
    R.sort_indices()
    hot = HotStepConfig(embed_size=c["d"], n_layers=c["n_layers"], head_num=c["head_num"], id_cat_rate=c["id_cat_rate"],
                        model_cat_rate=c["model_cat_rate"], drop_rate=c["drop_rate"], tau=c["tau"], cl_rate=c["cl_rate"],
                        emb_decay=c["emb_decay"], feat_reg_decay=c["feat_reg_decay"], batch_size=c["B"], lr=c["lr"], proj_impl=proj_impl)
    hp = gan.GanHyper(gp_rate=c["gp_rate"], G_rate=c["G_rate"], D_lr=c["D_lr"], log_log_scale=c["log_log_scale"],
                      real_data_tau=c["real_data_tau"], ui_pre_scale=c["ui_pre_scale"])
    cfg = FullStepConfig(hot=hot, gan=hp, m_topk_rate=c["m_topk_rate"], T=c["T"], G_drop1=c["G_drop1"], G_drop2=c["G_drop2"])
    P = {k[3:]: t(z[k]).contiguous() for k in z.files if k.startswith("G0/")}
    S = {k[3:]: t(z[k]) for k in z.files if k.startswith("D0/")}
    feats = (FeatureStore(t(z["image_feats"])), FeatureStore(t(z["text_feats"])))
    ui = BipartiteGraph.from_scipy(csr_norm(R), device=dev)
    iu = BipartiteGraph.from_scipy(csr_norm(R.T.tocsr()), device=dev)
    fs = FullStep(P, S, feats, t(R.indptr.astype(np.int64)), t(R.indices.astype(np.int64)), ui, iu, cfg, batch=c["B"])
    return fs, P, t


def run_and_check(dev="cuda", proj_impl="tc", steps=None):
    from mmssl_b200 import gan
    from mmssl_b200.engine import LIVE
    z, c = load_trace()
    fs, P, t = build(z, c, dev, proj_impl)
    n_steps = c["steps"] if steps is None else steps
    for s in range(n_steps):
        users, pos, neg = (t(z["sample"][s][j]) for j in range(3))
        out = fs.step(users, pos, neg,
                      model_masks=[t(z["mask_model"][4 * s + j]) for j in range(4)],
                      d_masks1=[t(z["mask_d1"][4 * s + j]) for j in range(4)],
                      d_masks2=[t(z["mask_d2"][4 * s + j]) for j in range(4)],
                      gumbel_u=t(z["gumbel_u"][s]), alpha=t(z["alpha"][s]).view(-1))
        # the five u_sim calls of the iteration, in the reference's order
        sims = list(fs.last["D_u_sim"]) + list(fs.last["G_u_sim"])
        for j, got in enumerate(sims):
            assert rel_err(got, torch.from_numpy(z["u_sim"][5 * s + j])) < TOL, (s, "u_sim", j)
        # Discriminator: penalty, gradients, state after Adam
        assert abs(float(out["gp"]) - float(z["gp"][s])) <= 2e-4 * abs(float(z["gp"][s])), (s, "gp")
        for k in gan.PARAMS:
            want = torch.from_numpy(z["Dgrad/" + k][s])
            got = out["D_grads"][k].cpu().view_as(want)
            if k in DEAD_BIAS:
                assert float(got.abs().max()) < 1e-5 * float(np.abs(z["Dgrad/" + DEAD_BIAS[k]][s]).max()), (s, k)
            else:
                assert rel_err(got, want) < 5e-4, (s, k, rel_err(got, want))
        for k in gan.PARAMS:
            if k not in DEAD_BIAS:
                assert rel_err(fs.D.t[k], torch.from_numpy(z["Dstate/" + k][s])) < 5e-4, (s, "Dstate", k)
        # generator: gradients of batch_loss (main.py:420) and parameters after AdamW
        for k in LIVE:
            e = rel_err(fs.hs.grads[k], torch.from_numpy(z["Ggrad/" + k][s]))
            assert e < TOL, (s, "Ggrad", k, e)
        for k in LIVE:
            e = rel_err(P[k], torch.from_numpy(z["Gparam/" + k][s]))
            assert e < TOL, (s, "Gparam", k, e)
    return fs


def _gemm_route():
    from mmssl_b200 import gan_ops
    return gan_ops.GEMM_IMPL


def regime_check(dev, m_topk_rate, T, proj_impl="simt"):
    """Regimes the recorded trace does not visit, against the oracle's FullStep (itself pinned to the trace at k = 4, T = 1):
    k = 0 (the reference's default rate at Baby: int(7050 * 1e-4) = 0 -> no pairs are ever collected, the modality graphs are
    empty from the third iteration on), T = 2 and T = 3 (pairs of several iterations accumulate before a rebuild, lists with
    duplicates).  Five iterations with generated draws; parameters of G after every iteration.  Discriminator: the gradients
    of every iteration against float64 from the device's own state and rows (d_step_vs_float64); its parameters after Adam
    only as a smoke check."""
    import scipy.sparse as sp  # noqa: F811
    from oracle import gan_oracle as GO, mmssl_oracle as O
    from mmssl_b200 import gan
    from mmssl_b200.engine import LIVE
    z, c = load_trace()
    c = dict(c, m_topk_rate=m_topk_rate, T=T)
    fs, P, t = build(z, c, dev, proj_impl=proj_impl)
    R = sp.csr_matrix((np.ones(len(z["train_rows"]), np.float32), (z["train_rows"], z["train_cols"])), shape=(c["U"], c["I"]))
    R.sort_indices()
    ocfg = O.HotPathConfig(embed_size=c["d"], n_layers=c["n_layers"], batch_size=c["B"], lr=c["lr"])
    gcfg = GO.GanConfig(m_topk_rate=m_topk_rate, T=T, D_lr=c["D_lr"], G_rate=c["G_rate"], gp_rate=c["gp_rate"])
    cpu = GO.FullStep({k[3:]: torch.from_numpy(z[k]).clone() for k in z.files if k.startswith("G0/")},
                      {k[3:]: torch.from_numpy(z[k]).clone() for k in z.files if k.startswith("D0/")},
                      torch.from_numpy(z["image_feats"]), torch.from_numpy(z["text_feats"]), R, ocfg, gcfg)
    g = torch.Generator().manual_seed(11)
    B, I, d = c["B"], c["I"], c["d"]
    mk = lambda n, w, p: ((torch.rand(n, w, generator=g) >= p) / (1 - p)).float()
    nnz_seen = []
    for s in range(5):
        users = torch.randperm(c["U"], generator=g)[:B]
        pos, neg = torch.randint(0, I, (B,), generator=g), torch.randint(0, I, (B,), generator=g)
        mm = [mk(I, d, c["drop_rate"]) for _ in range(4)]
        m1, m2 = [mk(2 * B, I // 4, 0.31) for _ in range(4)], [mk(2 * B, I // 8, 0.5) for _ in range(4)]
        gu, al = torch.rand(B, I, generator=g), torch.rand(2 * B, 1, generator=g)
        cpu.step(users.tolist(), pos.tolist(), neg.tolist(), mm, m1, m2, gu, al)
        on = lambda x: x.clone().to(dev)
        S0 = {k: v.detach().cpu().clone() for k, v in fs.D.t.items()}
        out = fs.step(on(users), on(pos), on(neg), model_masks=[on(m) for m in mm], d_masks1=[on(m) for m in m1],
                      d_masks2=[on(m) for m in m2], gumbel_u=on(gu), alpha=on(al.view(-1)))
        d_step_vs_float64(S0, dict(gp=out["gp"], grads=out["D_grads"]), *fs.last["D_u_sim"], users, R, gu, al, m1, m2, gcfg,
                          FP64_FLOOR[_gemm_route()], what=f"iteration {s}")
        nnz_seen.append(fs.hs.graphs[2].nnz)
        for k in LIVE:
            assert rel_err(P[k], cpu.P[k]) < 1e-4, (s, k, rel_err(P[k], cpu.P[k]))
        for k in gan.PARAMS:
            if k not in DEAD_BIAS:
                assert rel_err(fs.D.t[k], cpu.S[k]) < 5e-4, (s, k)
    k_top = int(I * m_topk_rate)
    if k_top == 0:
        assert nnz_seen[0] > 0 and nnz_seen[1:] == [0, 0, 0, 0] and fs.steady()
    else:          # rebuilds at iterations T, 2T, ...: the first one sees T iterations' worth of pairs
        assert nnz_seen[T] == T * B * k_top


def random_problem_check(dev, d=128, U=150, I=97, B=24, n_layers=3, m_topk_rate=0.04, steps=3, proj_impl="simt",
                         d_state_check=True):
    """A problem that shares nothing with the recorded trace -- other embedding width (other kernel instantiations), item count
    not a multiple of 8 (Discriminator widths int(I/4), int(I/8)), 3 GCN layers -- product FullStep vs the oracle's FullStep.
    Discriminator parity is its gradients of every iteration against float64 from the device's own state and rows
    (d_step_vs_float64); its parameters after Adam are a smoke check (``d_state_check``), because Adam's m / (sqrt(v) + eps)
    turns a last-bit difference of a gradient entry near zero into a difference of size lr (DESIGN section 2).
    Returns the FullStep and the distances of the first iteration's D step."""
    import scipy.sparse as sp  # noqa: F811
    from oracle import gan_oracle as GO, mmssl_oracle as O
    from mmssl_b200 import gan
    from mmssl_b200.engine import LIVE, FeatureStore
    from mmssl_b200.fullstep import FullStep, FullStepConfig
    from mmssl_b200.graph import BipartiteGraph
    from mmssl_b200.hotstep import HotStepConfig
    from mmssl_b200.synthetic import csr_norm, make_bipartite
    g = torch.Generator().manual_seed(d + I)
    R = make_bipartite(U, I, 6 * U, seed=d).tocsr().astype(np.float32)
    R.sort_indices()
    xav = lambda a, b: (torch.rand(a, b, generator=g) * 2 - 1) * (6.0 / (a + b)) ** 0.5
    dv, dt, h1, h2 = 20, 12, int(I / 4), int(I / 8)
    P = {"image_trans.weight": xav(d, dv), "image_trans.bias": torch.randn(d, generator=g) * 0.1, "text_trans.weight": xav(d, dt),
         "text_trans.bias": torch.randn(d, generator=g) * 0.1, "user_id_embedding.weight": xav(U, d), "item_id_embedding.weight": xav(I, d),
         "weight_dict.w_self_attention_cat": xav(4 * d, d), "weight_dict.w_q": xav(d, d), "weight_dict.w_k": xav(d, d)}
    kn = lambda o, i: torch.randn(o, i, generator=g) * (2.0 / i) ** 0.5
    S = {"net.0.weight": kn(h1, I), "net.0.bias": torch.zeros(h1), "net.2.weight": torch.ones(h1), "net.2.bias": torch.zeros(h1),
         "net.2.running_mean": torch.zeros(h1), "net.2.running_var": torch.ones(h1), "net.2.num_batches_tracked": torch.zeros((), dtype=torch.int64),
         "net.4.weight": kn(h2, h1), "net.4.bias": torch.zeros(h2), "net.6.weight": torch.ones(h2), "net.6.bias": torch.zeros(h2),
         "net.6.running_mean": torch.zeros(h2), "net.6.running_var": torch.ones(h2), "net.6.num_batches_tracked": torch.zeros((), dtype=torch.int64),
         "net.8.weight": kn(1, h2), "net.8.bias": torch.zeros(1)}
    feats = (torch.randn(I, dv, generator=g), torch.randn(I, dt, generator=g))
    ocfg = O.HotPathConfig(embed_size=d, n_layers=n_layers, batch_size=B)
    cpu = GO.FullStep({k: v.clone() for k, v in P.items()}, {k: v.clone() for k, v in S.items()}, feats[0], feats[1], R, ocfg,
                      GO.GanConfig(m_topk_rate=m_topk_rate))
    on = lambda x: x.clone().to(dev)
    Pd = {k: on(v).contiguous() for k, v in P.items()}
    cfg = FullStepConfig(hot=HotStepConfig(embed_size=d, n_layers=n_layers, batch_size=B, proj_impl=proj_impl), gan=gan.GanHyper(),
                         m_topk_rate=m_topk_rate)
    fs = FullStep(Pd, {k: on(v) for k, v in S.items()}, tuple(FeatureStore(on(f)) for f in feats), on(torch.from_numpy(R.indptr.astype(np.int64))),
                  on(torch.from_numpy(R.indices.astype(np.int64))), BipartiteGraph.from_scipy(csr_norm(R), device=dev),
                  BipartiteGraph.from_scipy(csr_norm(R.T.tocsr()), device=dev), cfg, batch=B)
    mk = lambda n, w, p: ((torch.rand(n, w, generator=g) >= p) / (1 - p)).float()
    first = None
    for s in range(steps):
        users = torch.randperm(U, generator=g)[:B]
        pos, neg = torch.randint(0, I, (B,), generator=g), torch.randint(0, I, (B,), generator=g)
        mm = [mk(I, d, 0.2) for _ in range(4)]
        m1, m2 = [mk(2 * B, h1, 0.31) for _ in range(4)], [mk(2 * B, h2, 0.5) for _ in range(4)]
        gu, al = torch.rand(B, I, generator=g), torch.rand(2 * B, 1, generator=g)
        cpu.step(users.tolist(), pos.tolist(), neg.tolist(), mm, m1, m2, gu, al)
        S0 = {k: v.detach().cpu().clone() for k, v in fs.D.t.items()}
        out = fs.step(on(users), on(pos), on(neg), model_masks=[on(m) for m in mm], d_masks1=[on(m) for m in m1],
                      d_masks2=[on(m) for m in m2], gumbel_u=on(gu), alpha=on(al.view(-1)))
        dist = d_step_vs_float64(S0, dict(gp=out["gp"], grads=out["D_grads"]), *fs.last["D_u_sim"], users, R, gu, al, m1, m2,
                                 GO.GanConfig(m_topk_rate=m_topk_rate), FP64_FLOOR[_gemm_route()], what=f"d={d} I={I} iteration {s}")
        first = dist if first is None else first
        for k in LIVE:
            assert rel_err(Pd[k], cpu.P[k]) < TOL, (s, k, rel_err(Pd[k], cpu.P[k]))
        if d_state_check:
            for k in gan.PARAMS:
                if k not in DEAD_BIAS:
                    assert rel_err(fs.D.t[k], cpu.S[k]) < 5e-4, (s, k, rel_err(fs.D.t[k], cpu.S[k]))
    return fs, first
