"""Full-size checks at the BASELINE shapes (Amazon-Baby / Amazon-Sports synthetic graphs):
size-independent properties of the SpMM operator pair and one full hot step against the CPU oracle."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from tests.golden_util import rel_err  # noqa: E402


@pytest.fixture(scope="module", params=["baby", "sports"])
def data(request):
    from mmssl_b200.graph import BipartiteGraph
    from mmssl_b200.synthetic import make_dataset
    ds = make_dataset(request.param)
    return ds, BipartiteGraph.from_scipy(ds.ui_norm), BipartiteGraph.from_scipy(ds.iu_norm)


def test_spmm_adjoint_linearity_softmax(data):
    from mmssl_b200 import ops
    ds, g_ui, g_iu = data
    d = ds.embed_size
    torch.manual_seed(0)
    for g, (m, n) in ((g_ui, (ds.n_users, ds.n_items)), (g_iu, (ds.n_items, ds.n_users))):
        x, x2, y = torch.randn(n, d, device="cuda"), torch.randn(n, d, device="cuda"), torch.randn(m, d, device="cuda")
        ax = ops.spmm(g.fwd, [x])[0]
        aty = ops.spmm(g.bwd, [y])[0]
        # <A x, y> == <x, A^T y>: the forward (CSR of A) and backward (CSR of A^T) operands describe the same matrix
        lhs, rhs = (ax.double() * y.double()).sum(), (x.double() * aty.double()).sum()
        assert abs(float(lhs - rhs)) < 1e-5 * abs(float(lhs)) + 1e-6
        # linearity, and the two-RHS launch equals two single launches
        both = ops.spmm(g.fwd, [x, x2])
        assert rel_err(both[0], ax) < 1e-6
        comb = ops.spmm(g.fwd, [2.0 * x - 0.5 * x2])[0]
        assert rel_err(comb, 2.0 * ax - 0.5 * both[1]) < 2e-5
        # softmax epilogue: every row is a distribution (rows without neighbours give 1/d)
        sm = ops.spmm(g.fwd, [x], epilogue=ops.EPI_SOFTMAX)[0]
        assert float((sm.sum(1) - 1).abs().max()) < 1e-5 and float(sm.min()) >= 0
        # exact row sums of the normalised graph: A 1 = sqrt(deg) (D^-1/2 R applied to ones)
        ones = torch.ones(n, d, device="cuda")
        deg = np.diff((ds.train if m == ds.n_users else ds.train.T.tocsr()).indptr)
        want = torch.from_numpy(np.sqrt(deg).astype(np.float32)).cuda()
        assert rel_err(ops.spmm(g.fwd, [ones])[0][:, 0], want) < 1e-5


def _random_modality_graphs(ds, n_edges, seed, device):
    """Distinct image / text graphs like the ones main.py:378-397 rebuilds: random (user, item) pairs, duplicates summed by
    scipy, csr_norm on each side.  Returns (scipy pairs for the oracle, BipartiteGraphs for the kernels)."""
    import scipy.sparse as sp
    from mmssl_b200.graph import BipartiteGraph
    from mmssl_b200.synthetic import csr_norm
    rng = np.random.default_rng(seed)
    out_sp, out_g = [], []
    for k in range(2):
        m = sp.csr_matrix((np.ones(n_edges, np.float32), (rng.integers(0, ds.n_users, n_edges), rng.integers(0, ds.n_items, n_edges))),
                          shape=(ds.n_users, ds.n_items))
        a, b = csr_norm(m), csr_norm(m.T.tocsr())
        out_sp += [a, b]
        out_g += [BipartiteGraph.from_scipy(a, device=device), BipartiteGraph.from_scipy(b, device=device)]
    return out_sp, out_g


def _empty_graph(shape, device):
    from mmssl_b200.graph import BipartiteGraph
    e = torch.zeros(0, dtype=torch.int64, device=device)
    return BipartiteGraph(e, e, torch.zeros(0, device=device), shape)


@pytest.mark.parametrize("name,modal,batch", [("baby", "alias", 1024), ("tiktok", "alias", 1024), ("tiktok", "distinct", 1024),
                                              ("tiktok", "empty", 1024), ("sports", "alias", 1024), ("sports", "distinct", 2048)])
def test_full_size_hot_step_vs_oracle(name, modal, batch):
    """One hot step at the BASELINE shapes -- Tiktok (9319 x 6710, V128/T768), Baby (19445 x 7050, V4096/T1024), Sports
    (35598 x 18357, K = 3: --weight_size [64,64,64], Models.py:201-211) -- with the three states of the modality graphs
    (alias of ui/iu at step 0, main.py:68-69; rebuilt distinct graphs with duplicate entries, main.py:378-397; empty, the steady
    state with the reference's default flags) and a batch beyond one 1024-block of the InfoNCE (main.py:228-246): the five loss
    terms and every live parameter gradient against the CPU oracle (pinned to the unmodified reference), 1e-4."""
    import bench
    from oracle import mmssl_oracle as O
    from mmssl_b200.engine import LIVE
    from mmssl_b200.hotstep import HotStep, HotStepConfig
    from mmssl_b200.synthetic import TripleSampler
    torch.set_num_threads(8)         # torch's CPU sparse kernels collapse with more threads (tools/cpu_threads.py)
    dev = torch.device("cuda")
    ds, P, feats, graphs, feats_cpu = bench.build_problem(name, 2022, dev)
    ui, iu = O.to_torch_coo(ds.ui_norm), O.to_torch_coo(ds.iu_norm)
    ograph = [ui, iu, ui, iu, ui, iu]
    graphs = list(graphs)
    if modal == "distinct":
        sps, gs = _random_modality_graphs(ds, 4 * batch, 11, dev)
        graphs[2:] = gs
        ograph[2:] = [O.to_torch_coo(m) for m in sps]
    elif modal == "empty":
        eu, ei = _empty_graph((ds.n_users, ds.n_items), dev), _empty_graph((ds.n_items, ds.n_users), dev)
        graphs[2:] = [eu, ei, eu, ei]
        z = lambda r, c: torch.sparse_coo_tensor(torch.zeros(2, 0, dtype=torch.int64), torch.zeros(0), (r, c))
        ograph[2:] = [z(ds.n_users, ds.n_items), z(ds.n_items, ds.n_users)] * 2
    cfg = HotStepConfig(embed_size=ds.embed_size, n_layers=ds.n_layers, batch_size=batch)
    hs = HotStep({k: v.clone() for k, v in P.items()}, feats, graphs, cfg, batch=batch, optimizer_step=False)
    g = torch.Generator().manual_seed(5)
    masks = tuple((torch.rand(ds.n_items, ds.embed_size, generator=g) >= 0.2).float() / 0.8 for _ in range(2))
    hs.masks = tuple(m.cuda() for m in masks)
    users, pos, neg = TripleSampler(ds.train, seed=3).sample(batch)
    hs.set_indices(users, pos, neg)
    out5 = hs.run().cpu()
    ocfg = O.HotPathConfig(embed_size=ds.embed_size, n_layers=ds.n_layers, batch_size=batch)
    po = {k: v.cpu().clone().requires_grad_(True) for k, v in P.items()}
    outs = O.forward_closed(po, feats_cpu[0], feats_cpu[1], tuple(ograph), ocfg, dropout_masks=masks)
    total, parts = O.hot_loss(outs, users, pos, neg, ds.n_items, ocfg)
    total.backward()
    for got, want in zip(out5.tolist(), [float(total), float(parts["mf"]), float(parts["emb"]), float(parts["feat_reg"]), float(parts["cl"])]):
        assert abs(got - want) <= 1e-4 * max(abs(want), 1e-12), (got, want)
    for k in LIVE:
        assert rel_err(hs.grads[k], po[k].grad) < 1e-4, (k, rel_err(hs.grads[k], po[k].grad))
