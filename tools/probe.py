"""GPU probe: in-graph (warm) latency of kernel chains at small scale, SpMM throughput at large scale.
Usage (on the GPU): python tools/probe.py [small] [large]"""
import json
import os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np, torch
from mmssl_b200 import ops
from mmssl_b200.graph import BipartiteGraph
from mmssl_b200.synthetic import make_dataset, make_bipartite, csr_norm

dev = torch.device("cuda")
PEAK = 3350.0      # GB/s: H100 SXM data-sheet HBM3 bandwidth (the fraction below is of the data sheet, not of a measured peak)


def graph_time(fn, reps=20, inner=1):
    """us per call of fn when `inner` calls are captured in a CUDA graph and replayed."""
    s = torch.cuda.Stream(); s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fn()
    torch.cuda.current_stream().wait_stream(s); torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(inner):
            fn()
    g.replay(); torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        g.replay()
    b.record(); torch.cuda.synchronize()
    return a.elapsed_time(b) * 1e3 / (reps * inner)


def cold_time(fn, flush, reps=5):
    ts = []
    for _ in range(reps):
        flush.add_(1.0)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record(); torch.cuda.synchronize()
        ts.append(a.elapsed_time(b) * 1e3)
    return sorted(ts)[len(ts) // 2]


def small(name):
    ds = make_dataset(name)
    d = ds.embed_size
    g_ui = BipartiteGraph.from_scipy(ds.ui_norm); g_iu = BipartiteGraph.from_scipy(ds.iu_norm)
    U, I = ds.n_users, ds.n_items
    xi = torch.randn(I, d, device=dev); yu = torch.empty(U, d, device=dev); yi = torch.empty(I, d, device=dev)
    x2 = torch.randn(I, 2 * d, device=dev); y2 = torch.empty(U, 2 * d, device=dev)
    out = {"config": name, "fwd_items": g_ui.fwd.desc.n_items, "iu_items": g_iu.fwd.desc.n_items,
           "ui_split_rows": g_ui.fwd.n_split_rows, "iu_split_rows": g_iu.fwd.n_split_rows}

    def chain():
        ops.spmm(g_ui.fwd, [xi], [yu]); ops.spmm(g_iu.fwd, [yu], [yi])
    out["spmm_pair_in_graph_us"] = graph_time(chain, inner=10)
    out["spmm_ui_in_graph_us"] = graph_time(lambda: ops.spmm(g_ui.fwd, [xi], [yu]), inner=20)
    out["spmm_iu_in_graph_us"] = graph_time(lambda: ops.spmm(g_iu.fwd, [yu], [yi]), inner=20)
    out["spmm_ui_2rhs_in_graph_us"] = graph_time(lambda: ops.spmm(g_ui.fwd, [x2[:, :d], x2[:, d:]], [y2[:, :d], y2[:, d:]]), inner=20)
    for impl in (0, 4, 8, 12, 16, 20, 24):
        out[f"ui_impl{impl}_us"] = round(graph_time(lambda: ops.spmm(g_ui.fwd, [xi], [yu], impl=impl), inner=20), 2)
        out[f"iu_impl{impl}_us"] = round(graph_time(lambda: ops.spmm(g_iu.fwd, [yu], [yi], impl=impl), inner=20), 2)
        out[f"ui2_impl{impl}_us"] = round(graph_time(lambda: ops.spmm(g_ui.fwd, [x2[:, :d], x2[:, d:]], [y2[:, :d], y2[:, d:]], impl=impl), inner=20), 2)
    # the GCN-layer forms of the call (epilogue operands indexed by the row): default vs early prefetch (impl bit 6)
    su = torch.zeros(U, d, device=dev); cu = torch.randn(U, d, device=dev); ysv = torch.softmax(torch.randn(U, d, device=dev), -1)
    for impl in (4, 68, 16, 80):
        out[f"gcn_fwd_impl{impl}_us"] = round(graph_time(lambda: ops.spmm(g_ui.fwd, [xi], [yu], epilogue=ops.EPI_SOFTMAX, ss=[su], s_mode=1,
                                                                          impl=impl), inner=20), 2)
        out[f"gcn_bwd_impl{impl}_us"] = round(graph_time(lambda: ops.spmm(g_iu.bwd, [xi], [yu], cs=[cu], alpha=0.33, epilogue=ops.EPI_SOFTMAX_BWD,
                                                                          ysaved=[ysv], impl=impl), inner=20), 2)
    # bulk-copy gather pipeline (csrc/spmm_bulk.cu): ring stages x warps per block x buckets per warp
    B = ops.SPMM_IMPL_BULK
    for wpb, tpw, tma in ((2, 1, 0), (4, 1, 0), (8, 1, 0), (4, 2, 0), (8, 2, 0), (2, 1, 1), (4, 1, 1), (8, 1, 1), (4, 2, 1)):
        for _ in (0,):
            for _ in (0,):
                v = B | (wpb << 4) | (tpw << 8) | (ops.SPMM_BULK_TMA if tma else 0)
                tag = f"bulk_w{wpb}t{tpw}" + ("_tma" if tma else "")
                out[f"ui_{tag}_us"] = round(graph_time(lambda: ops.spmm(g_ui.fwd, [xi], [yu], impl=v), inner=20), 2)
                out[f"iu_{tag}_us"] = round(graph_time(lambda: ops.spmm(g_iu.fwd, [yu], [yi], impl=v), inner=20), 2)
                out[f"ui2_{tag}_us"] = round(graph_time(lambda: ops.spmm(g_ui.fwd, [x2[:, :d], x2[:, d:]], [y2[:, :d], y2[:, d:]], impl=v), inner=20), 2)
    for v, tag in ((B, "bulk_auto"), (B | ops.SPMM_BULK_TMA, "bulk_tma")):
        out[f"gcn_fwd_{tag}_us"] = round(graph_time(lambda: ops.spmm(g_ui.fwd, [xi], [yu], epilogue=ops.EPI_SOFTMAX, ss=[su], s_mode=1, impl=v), inner=20), 2)
        out[f"gcn_bwd_{tag}_us"] = round(graph_time(lambda: ops.spmm(g_iu.bwd, [xi], [yu], cs=[cu], alpha=0.33, epilogue=ops.EPI_SOFTMAX_BWD,
                                                                         ysaved=[ysv], impl=v), inner=20), 2)
    yb = ops.spmm(g_ui.fwd, [xi], impl=B)[0]; ya = ops.spmm(g_ui.fwd, [xi], impl=0)[0]
    out["bulk_vs_ldg_max_abs_diff"] = float((ya - yb).abs().max())
    out["axpby_in_graph_us"] = graph_time(lambda: ops.axpby(xi, 1.0, 0.0, yi), inner=40)     # ~launch floor
    flush = torch.empty(192 * 1024 * 1024 // 4, device=dev)
    out["spmm_ui_cold_us"] = cold_time(lambda: ops.spmm(g_ui.fwd, [xi], [yu]), flush)
    out["spmm_iu_cold_us"] = cold_time(lambda: ops.spmm(g_iu.fwd, [yu], [yi]), flush)
    out["bulk_ui_cold_us"] = cold_time(lambda: ops.spmm(g_ui.fwd, [xi], [yu], impl=B), flush)
    out["bulk_iu_cold_us"] = cold_time(lambda: ops.spmm(g_iu.fwd, [yu], [yi], impl=B), flush)
    print(json.dumps(out))


def large(U, I, nnz, d, tag):
    t0 = time.time()
    r = make_bipartite(U, I, nnz, seed=1)
    a_ui, a_iu = csr_norm(r), csr_norm(r.T.tocsr())
    g_ui = BipartiteGraph.from_scipy(a_ui); g_iu = BipartiteGraph.from_scipy(a_iu)
    gen_s = time.time() - t0
    xi = torch.randn(I, d, device=dev); yu = torch.empty(U, d, device=dev); yi = torch.empty(I, d, device=dev)
    res = {"config": tag, "U": U, "I": I, "nnz": nnz, "d": d, "gen_s": round(gen_s, 1),
           "ui_items": g_ui.fwd.desc.n_items, "iu_items": g_iu.fwd.desc.n_items, "iu_split_rows": g_iu.fwd.n_split_rows}
    flush = torch.empty(192 * 1024 * 1024 // 4, device=dev)
    impl = int(os.environ.get("SPMM_IMPL", "0"))
    res["impl"] = impl
    for nm, g, x, y, M, N in (("ui", g_ui.fwd, xi, yu, U, I), ("iu", g_iu.fwd, yu, yi, I, U),
                              ("uiT", g_ui.bwd, yu, yi, I, U), ("iuT", g_iu.bwd, yi, yu, U, I)):
        ops.spmm(g, [x], [y], impl=impl); torch.cuda.synchronize()
        us = cold_time(lambda: ops.spmm(g, [x], [y], impl=impl), flush)
        if impl == 1:
            res[nm + "_hot_frac"] = round(g.hot_edge_fraction, 3)
        alg = 8 * nnz + 4 * (M + 1) + 4 * d * N + 4 * d * M
        gat = 8 * nnz + 4 * (M + 1) + 4 * d * nnz + 4 * d * M
        res[nm] = {"us": round(us, 1), "alg_MB": round(alg / 1e6, 1), "GBs": round(alg / us / 1e3, 1),
                   "frac": round(alg / us / 1e3 / PEAK, 3), "gather_GBs": round(gat / us / 1e3, 1)}
    # LDG kernel with residency hints: 16 = register-capped policy variant (the default here), +128 L2 streams, +256 L1 hot / cold rows
    for v in (16, 16 | 128):
        r = {}
        for nm, g, x, y in (("ui", g_ui.fwd, xi, yu), ("iu", g_iu.fwd, yu, yi), ("uiT", g_ui.bwd, yu, yi), ("iuT", g_iu.bwd, yi, yu)):
            ops.spmm(g, [x], [y], impl=v); torch.cuda.synchronize()
            r[nm] = round(cold_time(lambda: ops.spmm(g, [x], [y], impl=v), flush, reps=5), 1)
        res[f"ldg_impl{v}_us"] = r
    ya = ops.spmm(g_ui.fwd, [xi], impl=16)[0]
    for v in (16 | 128,):
        res[f"impl{v}_max_abs_diff"] = float((ya - ops.spmm(g_ui.fwd, [xi], impl=v)[0]).abs().max())
    res["hot_flag_fraction_ui"] = getattr(g_ui.fwd, "hot_flag_fraction", None)
    B = ops.SPMM_IMPL_BULK
    if os.environ.get("PROBE_BULK", "1") == "1":
        for tma in (0, 1):
            for wpb in (4, 8):
                for tpw in (1, 4):
                    v = B | (wpb << 4) | (tpw << 8) | (ops.SPMM_BULK_TMA if tma else 0)
                    nst = "tma" if tma else "ldgsts"
                    r = {}
                    for nm, g, x, y in (("ui", g_ui.fwd, xi, yu), ("iu", g_iu.fwd, yu, yi)):
                        ops.spmm(g, [x], [y], impl=v); torch.cuda.synchronize()
                        r[nm] = round(cold_time(lambda: ops.spmm(g, [x], [y], impl=v), flush, reps=3), 1)
                    res[f"bulk_{nst}_w{wpb}t{tpw}_us"] = r
        ya = ops.spmm(g_ui.fwd, [xi], impl=0)[0]; yb = ops.spmm(g_ui.fwd, [xi], impl=B)[0]
        res["bulk_vs_ldg_max_abs_diff"] = float((ya - yb).abs().max())
    print(json.dumps(res))


if __name__ == "__main__":
    which = sys.argv[1:] or ["small"]
    if "small" in which:
        small("baby"); small("sports")
    if "large" in which:
        large(1_000_000, 200_000, 20_000_000, 128, "syn1m")
    if "mid" in which:
        large(200_000, 50_000, 4_000_000, 64, "mid-d64")


def kernels(name="baby"):
    """Isolated in-graph latency of the small kernels on the main-stream critical path."""
    ds = make_dataset(name)
    d, U, I = ds.embed_size, ds.n_users, ds.n_items
    f = dict(device=dev)
    ya, e, g = torch.randn(U, d, **f), torch.randn(U, d, **f), torch.randn(U, d, **f)
    wcat = torch.randn(4 * d, d, **f) * 0.1
    w, w_t = ops.wsum(wcat, d, 4)
    out = {"config": name}
    out["id_fuse2_fwd_U_us"] = round(graph_time(lambda: ops.id_fuse2_fwd(ya, None, 1.0, w, e, 0.36), inner=10), 2)
    o, zn, nrm = ops.id_fuse2_fwd(ya, None, 1.0, w, e, 0.36)
    out["id_fuse2_bwd_U_us"] = round(graph_time(lambda: ops.id_fuse2_bwd(g, zn, nrm, ya, None, 1.0, w_t, 0.36, None, None, False), inner=10), 2)
    _, _, pu = ops.id_fuse2_bwd(g, zn, nrm, ya, None, 1.0, w_t, 0.36, None, None, False)
    dw = torch.empty(4 * d, d, **f)
    out["dwcat_reduce_us"] = round(graph_time(lambda: ops.dwcat_reduce(pu, pu[:111], d, 4, dw), inner=10), 2)
    B = 1024
    users = torch.randperm(U, device=dev)[:B]; pos = torch.randint(0, I, (B,), device=dev); neg = torch.randint(0, I, (B,), device=dev)
    uf, itf = torch.randn(U, d, **f), torch.randn(I, d, **f)
    gu, gi = torch.zeros(U, d, **f), torch.zeros(I, d, **f)
    part = torch.empty(2 * 64, **f)
    out["bpr_us"] = round(graph_time(lambda: ops.bpr(uf, itf, itf, users, pos, neg, mode=3, reg_coef=1e-8, part=part, g_u=gu, g_p=gi, g_n=gi), inner=10), 2)
    seed = torch.ones(1, **f)
    for impl in ("auto", "simt"):      # auto = tensor cores at this size (csrc/loss_tc.cu)
        wk = ops.InfoNCEWork(B, d, dev, impl=impl)
        tag = "tc" if wk.tc else "simt"
        out[f"nce_fwd_{tag}_us"] = round(graph_time(lambda: ops.infonce_forward(ya, uf, users, 2.0, wk, g_loss=seed), inner=10), 2)
        out[f"nce_bwd_{tag}_us"] = round(graph_time(lambda: ops.infonce_backward(users, 2.0, wk, gu, gu), inner=10), 2)
    s = torch.randn(U, d, **f); a2 = torch.randn(U, 2 * d, **f); o2 = torch.empty(U, d, **f)
    out["combine_fwd_us"] = round(graph_time(lambda: ops.combine_fwd(s, a2[:, :d], a2[:, d:], 1 / 3, 0.55, o2), inner=10), 2)
    out["fill_us"] = round(graph_time(lambda: gu.zero_(), inner=20), 2)
    print(json.dumps(out))


def pipe(name="baby"):
    """The software-pipelined SpMM walk (impl bit 9) against the one-item-per-group kernel at small scale: plain products,
    two right-hand sides, the GCN-layer forms; grid sizes from 2 to 8 blocks per SM."""
    ds = make_dataset(name)
    d = ds.embed_size
    g_ui = BipartiteGraph.from_scipy(ds.ui_norm); g_iu = BipartiteGraph.from_scipy(ds.iu_norm)
    U, I = ds.n_users, ds.n_items
    xi = torch.randn(I, d, device=dev); yu = torch.empty(U, d, device=dev); yi = torch.empty(I, d, device=dev)
    x2 = torch.randn(I, 2 * d, device=dev); y2 = torch.empty(U, 2 * d, device=dev)
    su = torch.zeros(U, d, device=dev); cu = torch.randn(U, d, device=dev); ysv = torch.softmax(torch.randn(U, d, device=dev), -1)
    out = {"config": name, "ui_items": g_ui.fwd.desc.n_items, "iu_items": g_iu.fwd.desc.n_items}

    def forms(impl):
        return {"ui": round(graph_time(lambda: ops.spmm(g_ui.fwd, [xi], [yu], impl=impl), inner=20), 2),
                "iu": round(graph_time(lambda: ops.spmm(g_iu.fwd, [yu], [yi], impl=impl), inner=20), 2),
                "ui2": round(graph_time(lambda: ops.spmm(g_ui.fwd, [x2[:, :d], x2[:, d:]], [y2[:, :d], y2[:, d:]], impl=impl), inner=20), 2),
                "gcn_fwd": round(graph_time(lambda: ops.spmm(g_ui.fwd, [xi], [yu], epilogue=ops.EPI_SOFTMAX, ss=[su], s_mode=1, impl=impl), inner=20), 2),
                "gcn_bwd": round(graph_time(lambda: ops.spmm(g_iu.bwd, [xi], [yu], cs=[cu], alpha=0.33, epilogue=ops.EPI_SOFTMAX_BWD,
                                                             ysaved=[ysv], impl=impl), inner=20), 2)}
    for impl in (4, 6, 2):
        out[f"impl{impl}"] = forms(impl)
    for per_sm in (0, 2, 3, 4, 6, 8):
        ops.spmm_pipe_set_blocks(per_sm * torch.cuda.get_device_properties(0).multi_processor_count)
        for pre in (0, 64):
            out[f"pipe_b{per_sm}_pre{pre}"] = forms(ops.SPMM_IMPL_PIPE | pre)
    ops.spmm_pipe_set_blocks(0)
    ya = ops.spmm(g_ui.fwd, [xi], impl=4)[0]; yb = ops.spmm(g_ui.fwd, [xi], impl=ops.SPMM_IMPL_PIPE)[0]
    out["pipe_vs_default_max_abs_diff"] = float((ya - yb).abs().max())
    print(json.dumps(out))


def plan(name="baby"):
    """Where the work plan cuts rows (ops.spmm_plan_set_cuts): the longest item is the kernel's critical path on a small graph."""
    ds = make_dataset(name)
    d = ds.embed_size
    U, I = ds.n_users, ds.n_items
    xi = torch.randn(I, d, device=dev); yu = torch.empty(U, d, device=dev); yi = torch.empty(I, d, device=dev)
    x2 = torch.randn(I, 2 * d, device=dev); y2 = torch.empty(U, 2 * d, device=dev)
    su = torch.zeros(U, d, device=dev); cu = torch.randn(U, d, device=dev); ysv = torch.softmax(torch.randn(U, d, device=dev), -1)
    out = {"config": name}
    ref = None
    for cuts in ((64, 32, 1024, 64), (48, 24, 1024, 64), (32, 32, 1024, 64), (32, 16, 1024, 64), (32, 16, 512, 32), (24, 12, 512, 32), (16, 16, 512, 32),
                 (16, 8, 512, 32), (8, 8, 256, 16)):
        ops.spmm_plan_set_cuts(*cuts)
        g_ui = BipartiteGraph.from_scipy(ds.ui_norm); g_iu = BipartiteGraph.from_scipy(ds.iu_norm)
        r = {"ui_items": g_ui.fwd.desc.n_items, "iu_items": g_iu.fwd.desc.n_items, "ui_split": g_ui.fwd.n_split_rows, "iu_split": g_iu.fwd.n_split_rows}
        for impl in (4, 68):
            r[f"impl{impl}"] = {
                "ui": round(graph_time(lambda: ops.spmm(g_ui.fwd, [xi], [yu], impl=impl), inner=20), 2),
                "iu": round(graph_time(lambda: ops.spmm(g_iu.fwd, [yu], [yi], impl=impl), inner=20), 2),
                "ui2": round(graph_time(lambda: ops.spmm(g_ui.fwd, [x2[:, :d], x2[:, d:]], [y2[:, :d], y2[:, d:]], impl=impl), inner=20), 2),
                "gcn_fwd": round(graph_time(lambda: ops.spmm(g_ui.fwd, [xi], [yu], epilogue=ops.EPI_SOFTMAX, ss=[su], s_mode=1, impl=impl), inner=20), 2),
                "gcn_bwd": round(graph_time(lambda: ops.spmm(g_iu.bwd, [xi], [yu], cs=[cu], alpha=0.33, epilogue=ops.EPI_SOFTMAX_BWD,
                                                             ysaved=[ysv], impl=impl), inner=20), 2)}
        y = ops.spmm(g_ui.fwd, [xi], impl=4)[0]
        if ref is None:
            ref = y.clone()
        r["max_abs_diff_vs_first"] = float((y - ref).abs().max())
        out["cuts_%d_%d_%d_%d" % cuts] = r
    ops.spmm_plan_set_cuts(64, 32, 1024, 64)
    print(json.dumps(out))


if __name__ == "__main__" and "plan" in sys.argv[1:]:
    plan("baby"); plan("sports")
    sys.exit(0)

if __name__ == "__main__" and "pipe" in sys.argv[1:]:
    pipe("baby"); pipe("sports")
    sys.exit(0)

if __name__ == "__main__" and "kernels" in sys.argv[1:]:
    kernels("baby")
