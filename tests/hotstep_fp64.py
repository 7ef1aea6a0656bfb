"""Float64 yardstick of the training hot step (``mmssl_b200.hotstep.HotStep``), shared by tests/test_gpu_zz_hotstep_fp64.py and
its emulator twin tests/test_emu_hotstep_fp64.py.  A helper, not a test file.

What is compared: the five loss values, the forward outputs and the seven live parameter gradients of one device step with
``oracle.mmssl_oracle.forward_closed`` + ``hot_loss`` + autograd evaluated in float64 on the same inputs (parameters,
features, masks and graph values are the fp32 numbers the device gets, cast up).  The same oracle in float32 sets the bound:

    a device result may be ``K_FP32`` times as far from float64 as fp32 autograd is, and never has to be closer than a
    floor stated per route (``FLOOR``).

Three measures, because max|a-b| / max|b| alone lets one large row hide the others:
  norm      max|a-b| / max|b|                                       (every tensor)
  row       max over rows of ||row(a) - row(b)|| / ||row(b)||, rows with ||row(b)|| > ROW_TINY * the largest row norm
  row/<class>  the same maximum over one class of rows of the two embedding-table gradients: rows in / outside the batch,
            positives / negatives / untouched items, rows the SpMM plan splits or treats as heavy, the last partial
            128-row tile.
"""
from __future__ import annotations

import contextlib
from dataclasses import dataclass, field, replace
from typing import Dict, Optional, Tuple

import numpy as np
import scipy.sparse as sp
import torch

from oracle import mmssl_oracle as O

LIVE = ("image_trans.weight", "image_trans.bias", "text_trans.weight", "text_trans.bias",
        "user_id_embedding.weight", "item_id_embedding.weight", "weight_dict.w_self_attention_cat")
P_EU, P_EI = LIVE[4], LIVE[5]
LOSSES = ("total", "mf", "emb", "feat_reg", "cl")
OUTS = ("u_f", "i_f", "i_v", "i_t", "u_v", "u_t", "u_vid", "u_tid", "i_vid", "i_tid")     # Engine.forward's ten (12 less the two repeats)
OUT_OF_12 = (0, 1, 2, 3, 4, 5, 8, 9, 10, 11)
DEFAULT_CUTS = (64, 32, 1024, 64)      # csrc/graph.cu: split threshold, segment, heavy threshold, heavy segment
K_FP32 = 4.0
ROW_TINY = 1e-6
# A route is "<projection>/<InfoNCE>": projection 'simt' (fp32 CUDA cores) or 'tc' (bf16 hi/lo on tensor cores), InfoNCE 'simt' or
# 'auto' (tensor cores where n <= 2048 and d in {64, 128}).
# Floors, from the largest distances tests/test_gpu_zz_hotstep_fp64.py saw where the 4x rule alone did not cover them
# (NVIDIA H100 80GB HBM3, power limit 700 W), with about 2x headroom:
#   * CUDA-core projection, either InfoNCE: nothing exceeded 4x fp32 autograd (largest device figures 4.3e-6 norm-wise, 1.1e-5
#     row-wise where fp32 autograd itself is at 8.7e-5, losses 1.1e-6), so the floors are the 1e-5 an all-fp32 route should hold.
#   * tensor-core projection: a bf16 hi/lo pair carries 2^-17 = 7.6e-6 per operand, relative to the operand's largest entry, so
#     X = F W^T and what is propagated from it sit at 6.6e-6 norm-wise / 1.0e-5 row-wise; dW = (gX * mask)^T F is a second such
#     product of an operand that already carries the first one's error: 1.14e-5 norm-wise; and because the error scales with the
#     largest entry of the product, not with the row, rows of dW with a small norm reach 3.97e-5.  feat_reg, a sum of squares
#     of those outputs, is 7.05e-6 off (twice the outputs' error).  Hence 2.5e-5 / 8e-5 / 1.5e-5.
FLOOR: Dict[str, Dict[str, float]] = {
    "simt/simt": dict(norm=1e-5, row=1e-5, loss=2e-6),
    "simt/auto": dict(norm=1e-5, row=1e-5, loss=2e-6),
    "tc/simt": dict(norm=2.5e-5, row=8e-5, loss=1.5e-5),
    "tc/auto": dict(norm=2.5e-5, row=8e-5, loss=1.5e-5),
}
# (route, tensor, measure) -> (largest device distance, largest fp32-autograd distance) seen by assert_close in this process
LEDGER: Dict[Tuple[str, str, str], Tuple[float, float]] = {}


# ---------------------------------------------------------------------------------------------------------------- problem
@dataclass
class Problem:
    U: int
    I: int
    d: int
    dv: int
    dt: int
    modal: str
    cuts: Tuple[int, int, int, int]
    train: sp.csr_matrix                      # raw interactions
    coo: list                                 # six (rows, cols, fp32 vals, shape); aliased entries are the same object
    params: Dict[str, torch.Tensor]
    feats: Tuple[torch.Tensor, torch.Tensor]
    masks: Tuple[torch.Tensor, torch.Tensor]
    users: torch.Tensor
    pos: torch.Tensor
    neg: torch.Tensor
    _dense: dict = field(default_factory=dict)

    def sparse(self, dtype):
        """The six graphs as torch sparse COO tensors in `dtype` (the fp32 values cast, duplicates kept)."""
        if dtype not in self._dense:
            made = {}
            for g in self.coo:
                if id(g) not in made:
                    r, c, v, shape = g
                    idx = torch.from_numpy(np.vstack((r, c)).astype(np.int64))
                    made[id(g)] = torch.sparse_coo_tensor(idx, torch.from_numpy(v).to(dtype), shape)
            self._dense[dtype] = [made[id(g)] for g in self.coo]
        return self._dense[dtype]

    def with_batch(self, users, pos, neg, masks=None):
        t = lambda x: torch.as_tensor(np.asarray(x), dtype=torch.int64)
        return replace(self, users=t(users), pos=t(pos), neg=t(neg), masks=self.masks if masks is None else masks)


def train_matrix(U, I, seed, cuts=DEFAULT_CUTS):
    """Interactions with every class of row: user 0 / item 0 over the heavy threshold (when the other side is large enough),
    users and items 1..3 over the split threshold, user U - 2 and item I - 2 without any edge."""
    from mmssl_b200.synthetic import make_bipartite
    R = make_bipartite(U, I, 6 * U, seed=seed).toarray() > 0
    rng = np.random.default_rng(seed + 1)
    split, _, heavy, _ = cuts
    if I >= heavy + 16:
        R[0, rng.choice(I, heavy + 6, replace=False)] = True
    if U >= heavy + 16:
        R[rng.choice(U, heavy + 6, replace=False), 0] = True
    for j in (1, 2, 3):
        R[j, rng.choice(I, min(split + 4 + j, I // 2), replace=False)] = True
        R[rng.choice(U, min(split + 4 + j, U // 2), replace=False), j] = True
    R[U - 2, :] = False
    R[:, I - 2] = False
    return sp.csr_matrix(R.astype(np.float32))


def _norm_coo(mat, duplicates=False):
    from mmssl_b200.synthetic import csr_norm
    m = csr_norm(mat).tocoo()
    r, c, v = m.row.astype(np.int64), m.col.astype(np.int64), m.data.astype(np.float32)
    if duplicates and len(v):       # every third entry stored as two halves: exact in fp32, uncoalesced like the rebuilt graphs
        k = np.arange(0, len(v), 3)
        v = v.copy()
        v[k] *= np.float32(0.5)
        r, c, v = np.concatenate((r, r[k])), np.concatenate((c, c[k])), np.concatenate((v, v[k]))
        order = np.random.default_rng(len(v)).permutation(len(v))
        r, c, v = r[order], c[order], v[order]
    return (r, c, v, tuple(mat.shape))


def problem(U, I, d=64, B=96, modal="alias", dv=72, dt=40, head_num=4, seed=0, cuts=DEFAULT_CUTS, drop=0.2, train=None,
            table_scale=1.0) -> Problem:
    """A seeded problem: training graph (train_matrix, or `train`), the three states of the modality graphs ('alias': the
    training graph itself, 'distinct': four random graphs with duplicate COO entries, 'empty'), features, parameters with the
    reference's init (`table_scale` multiplies the two embedding tables), dropout masks and one sampled batch."""
    from mmssl_b200.synthetic import TripleSampler
    R = train_matrix(U, I, seed, cuts) if train is None else train
    ui, iu = _norm_coo(R), _norm_coo(R.T.tocsr())
    rng = np.random.default_rng(seed + 7)
    if modal == "alias":
        coo = [ui, iu, ui, iu, ui, iu]
    elif modal == "empty":
        e = np.zeros(0, np.int64)
        eu, ei = (e, e, np.zeros(0, np.float32), (U, I)), (e, e, np.zeros(0, np.float32), (I, U))
        coo = [ui, iu, eu, ei, eu, ei]
    else:
        def rand(shape, nnz):
            m = sp.csr_matrix((np.ones(nnz, np.float32), (rng.integers(0, shape[0], nnz), rng.integers(0, shape[1], nnz))), shape=shape)
            return _norm_coo(m, duplicates=True)
        coo = [ui, iu, rand((U, I), 3 * U), rand((I, U), 2 * U + 5), rand((U, I), 2 * U), rand((I, U), U + 3)]
    cfg = O.HotPathConfig(embed_size=d, head_num=head_num)
    params = O.init_params(U, I, dv, dt, cfg, seed=seed)
    if table_scale != 1.0:
        params[P_EU] = params[P_EU] * table_scale
        params[P_EI] = params[P_EI] * table_scale
    g = torch.Generator().manual_seed(seed)
    feats = (torch.randn(I, dv, generator=g), torch.randn(I, dt, generator=g))
    p = Problem(U, I, d, dv, dt, modal, tuple(cuts), R.tocsr(), coo, params, feats, new_masks(I, d, drop, g), None, None, None)
    return p.with_batch(*TripleSampler(R.tocsr(), seed=seed + 3).sample(B))


def new_masks(I, d, drop, gen):
    keep = 1.0 - drop if drop > 0 else 1.0
    return tuple((torch.rand(I, d, generator=gen) >= (drop if drop > 0 else -1.0)).float() / keep for _ in range(2))


# ---------------------------------------------------------------------------------------------------------------- reference
def oracle_cfg(cfg) -> O.HotPathConfig:
    return O.HotPathConfig(embed_size=cfg.embed_size, n_layers=cfg.n_layers, head_num=cfg.head_num, id_cat_rate=cfg.id_cat_rate,
                           model_cat_rate=cfg.model_cat_rate, drop_rate=cfg.drop_rate, tau=cfg.tau, cl_rate=cfg.cl_rate,
                           emb_decay=cfg.emb_decay, feat_reg_decay=cfg.feat_reg_decay, batch_size=cfg.batch_size)


def reference(p: Problem, cfg, dtype, params=None, training=True):
    """forward_closed + hot_loss + backward of the oracle in `dtype` on problem `p` (cfg: a HotStepConfig); `params` replaces
    the problem's parameters (fp32 values, e.g. a device state copied back).  Returns dict(losses [5], outs (12), grads {7})."""
    ocfg = oracle_cfg(cfg)
    src = p.params if params is None else params
    P = {k: v.detach().cpu().to(dtype).clone().requires_grad_(k in LIVE) for k, v in src.items()}
    use_masks = training and cfg.drop_rate > 0
    masks = tuple(m.to(dtype) for m in p.masks) if use_masks else None
    outs = O.forward_closed(P, p.feats[0].to(dtype), p.feats[1].to(dtype), p.sparse(dtype), ocfg, dropout_masks=masks, training=False)
    total, parts = O.hot_loss(outs, p.users, p.pos, p.neg, p.I, ocfg)
    total.backward()
    losses = torch.stack([total.detach()] + [torch.as_tensor(parts[k], dtype=dtype).detach() for k in LOSSES[1:]])
    zero = lambda k: torch.zeros_like(P[k])
    return dict(losses=losses, outs=tuple(o.detach() for o in outs),
                grads={k: (P[k].grad if P[k].grad is not None else zero(k)) for k in LIVE})


def both(p: Problem, cfg, params=None, training=True):
    return (reference(p, cfg, torch.float64, params, training), reference(p, cfg, torch.float32, params, training))


# ---------------------------------------------------------------------------------------------------------------- device
@contextlib.contextmanager
def nce_route(impl: str):
    """ops.NCE_IMPL is read when a HotStep allocates its InfoNCE work buffers: set around the construction, restored after."""
    from mmssl_b200 import ops
    old = ops.NCE_IMPL
    ops.NCE_IMPL = impl
    try:
        yield
    finally:
        ops.NCE_IMPL = old


def device_graphs(p: Problem):
    from mmssl_b200.graph import BipartiteGraph
    made = {}
    for g in p.coo:
        if id(g) not in made:
            r, c, v, shape = g
            made[id(g)] = BipartiteGraph(torch.from_numpy(r).cuda(), torch.from_numpy(c).cuda(), torch.from_numpy(v).cuda(), shape)
    return [made[id(g)] for g in p.coo]


def hot_step(p: Problem, cfg, route: str, optimizer_step=False, training=True, sampler=None, graphs=None):
    """The device HotStep of problem `p` on `route` ('<proj>/<nce>'), masks and batch set, not yet run."""
    from mmssl_b200.engine import FeatureStore
    from mmssl_b200.hotstep import HotStep
    proj, nce = route.split("/")
    cfg = replace(cfg, proj_impl=proj)
    P = {k: v.clone().cuda().contiguous() for k, v in p.params.items()}
    feats = tuple(FeatureStore(f.cuda()) for f in p.feats)
    with nce_route(nce):
        hs = HotStep(P, feats, device_graphs(p) if graphs is None else graphs, cfg, batch=int(p.users.numel()),
                     optimizer_step=optimizer_step, sampler=sampler)
    hs.training = training
    hs.masks = tuple(m.clone().cuda() for m in p.masks)
    hs.set_indices(p.users, p.pos, p.neg)
    return hs


# ---------------------------------------------------------------------------------------------------------------- measures
def row_classes(p: Problem) -> Dict[str, Dict[str, torch.Tensor]]:
    """Boolean row masks of the two embedding tables, by the way a row's gradient is produced."""
    split, _, heavy, _ = p.cuts
    deg_u, deg_i = np.zeros(p.U, np.int64), np.zeros(p.I, np.int64)
    seen = set()
    for r, c, v, shape in p.coo:       # a row's stored entries (duplicates counted) in A and, as a column, in A^T
        if id(r) in seen:
            continue
        seen.add(id(r))
        (by_row, by_col) = (deg_u, deg_i) if shape == (p.U, p.I) else (deg_i, deg_u)
        by_row[:] = np.maximum(by_row, np.bincount(r, minlength=len(by_row)))
        by_col[:] = np.maximum(by_col, np.bincount(c, minlength=len(by_col)))

    def member(n, idx):
        m = torch.zeros(n, dtype=torch.bool)
        m[idx] = True
        return m

    def common(n, deg):
        deg = torch.from_numpy(deg)
        return {"split": (deg > split) & (deg <= heavy), "heavy": deg > heavy, "last tile": torch.arange(n) >= n - n % 128}
    b = member(p.U, p.users)
    po, ne = member(p.I, p.pos), member(p.I, p.neg)
    return {P_EU: {"batch": b, "non-batch": ~b, **common(p.U, deg_u)},
            P_EI: {"positive": po, "negative": ne, "untouched": ~(po | ne), **common(p.I, deg_i)}}


def distances(a, b64, classes=None):
    """{measure: (distance, worst row or -1)} of `a` against the float64 tensor `b64`."""
    a, b = a.detach().double().cpu().reshape(b64.shape), b64.detach().double().cpu()
    diff = (a - b).abs()
    out = {"norm": (float(diff.max()) / max(float(b.abs().max()), 1e-300) if b.numel() else 0.0, -1)}
    if b.dim() != 2 or b.shape[0] < 2:
        return out
    nb = b.norm(dim=1)
    ok = nb > ROW_TINY * float(nb.max())
    rel = torch.where(ok, (a - b).norm(dim=1) / nb.clamp_min(1e-300), torch.zeros_like(nb))
    for name, m in [("row", torch.ones_like(ok))] + [("row/" + k, v) for k, v in (classes or {}).items()]:
        sel = rel * (m & ok)
        if bool((m & ok).any()):
            j = int(sel.argmax())
            out[name] = (float(sel[j]), j)
    return out


def assert_close(name, dev, f32, f64, route, classes=None, what=""):
    """`dev` within K_FP32 x the distance of `f32` (fp32 autograd) to `f64`, or the route's floor, on every measure."""
    assert bool(torch.isfinite(dev.detach().cpu()).all()), f"{what} {name}: non-finite device result"
    e_dev, e_32 = distances(dev, f64, classes), distances(f32, f64, classes)
    for m, (e, row) in e_dev.items():
        ref = e_32[m][0]
        key = (route, name, m)
        seen = LEDGER.get(key, (0.0, 0.0))
        LEDGER[key] = (max(seen[0], e), max(seen[1], ref))
        bound = max(K_FP32 * ref, FLOOR[route]["norm" if m == "norm" else "row"])
        assert e <= bound, (f"{what} [{route}] {name} {m}: device {e:.3g} from float64 (worst row {row}), fp32 autograd {ref:.3g}, "
                            f"bound {bound:.3g}")
    return e_dev


def assert_losses(dev5, f32, f64, route, what=""):
    dev5 = dev5.detach().double().cpu()
    assert bool(torch.isfinite(dev5).all()), f"{what}: non-finite loss {dev5.tolist()}"
    for j, name in enumerate(LOSSES):
        want, lo, got = float(f64[j]), float(f32[j]), float(dev5[j])
        if want == 0.0:
            assert got == 0.0, f"{what} loss {name}: {got} where float64 gives exactly 0"
            continue
        e, ref = abs(got - want) / abs(want), abs(lo - want) / abs(want)
        key = (route, "loss " + name, "rel")
        seen = LEDGER.get(key, (0.0, 0.0))
        LEDGER[key] = (max(seen[0], e), max(seen[1], ref))
        bound = max(K_FP32 * ref, FLOOR[route]["loss"])
        assert e <= bound, f"{what} [{route}] loss {name}: device {got!r}, float64 {want!r} ({e:.3g}), fp32 autograd {ref:.3g}, bound {bound:.3g}"


def check_step(hs, p: Problem, cfg, route, what="", out5=None, hi=None, lo=None, params=None, outs=False):
    """One device step (run here unless `out5` is given) against float64: five losses, seven gradients, optionally the outputs."""
    if hi is None:
        hi, lo = both(p, cfg, params, training=hs.training)
    if out5 is None:
        out5 = hs.run()
    assert_losses(out5, lo["losses"], hi["losses"], route, what)
    cls = row_classes(p)
    for k in LIVE:
        assert_close(k, hs.grads[k], lo["grads"][k], hi["grads"][k], route, cls.get(k), what)
    if outs:
        dev_outs, _ = hs.engine.forward(hs.P, hs.feats, hs.graphs, hs._masks)
        for name, j, got in zip(OUTS, OUT_OF_12, dev_outs):
            assert_close("out " + name, got, lo["outs"][j], hi["outs"][j], route, None, what)
    return hi, lo


def report() -> str:
    lines = [f"{r:10s} {t:42s} {m:16s} device {a:.3g}  fp32 {b:.3g}" for (r, t, m), (a, b) in sorted(LEDGER.items())]
    return "\n".join(lines)
