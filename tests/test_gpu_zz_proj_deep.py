"""The deep-ring instance of the grouped projection GEMM (csrc/proj_tc.cu, gemm_bf16x3_group_kernel<N, true>): one CTA per
SM with a 4-stage (N = 64) or 5-stage (N = 32) ring, selected when the grid is at most one CTA per SM, i.e. at the engine's
132-CTA cap.  Checked with the helpers of test_gpu_zz_proj_grouped.py at max_ctas = 132, and the hot step's dropout masks are
checked against a direct draw now that the step draws them beside the projection GEMM.  tests/test_emu_proj_deep.py runs the
same bodies at small sizes in the emulator."""
import pytest
import torch

from tests import test_gpu_zz_proj_grouped as G

pytestmark = pytest.mark.gpu

CAP = 132   # Engine.proj_max_ctas: one CTA per SM of the H100 SXM
SHAPES = [G.BABY_FWD, G.BABY_WGRAD, G.SPORTS_FWD, G.SPORTS_WGRAD]
IDS = ["baby_fwd", "baby_wgrad", "sports_fwd", "sports_wgrad"]


@pytest.mark.parametrize("shapes", SHAPES, ids=IDS)
def test_deep_bitwise_vs_single_kernel(shapes):
    G.check_group_bitwise_vs_single(shapes, CAP)


@pytest.mark.parametrize("shapes", SHAPES, ids=IDS)
def test_deep_vs_fp64(shapes):
    G.check_group_vs_fp64(shapes, CAP)


@pytest.mark.parametrize("shapes", SHAPES, ids=IDS)
def test_deep_plan(shapes):
    G.check_plan(shapes, CAP)


def _kernel_names(shapes, max_ctas):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        G._run_group(shapes, max_ctas)
    return [e.name for e in prof.events() if "gemm_bf16x3_group_kernel" in e.name]


@pytest.mark.parametrize("shapes", [
    [(5000, 32, 4096), (5000, 32, 1024)],        # N = 32: 5 stages
    [(7001, 64, 1000), (333, 64, 7050)],        # ragged M and K
    [(7050, 64, 4096)],                         # one problem
    [(5000, 128, 4096), (5000, 128, 1024)],     # N = 128: one CTA per SM already, the one instance
], ids=["n32", "ragged", "one_problem", "n128"])
def test_deep_shapes_and_instance(shapes):
    G.check_group_vs_fp64(shapes, CAP)
    G.check_plan(shapes, CAP)
    n = shapes[0][1]
    deep, full = _kernel_names(shapes, CAP), _kernel_names(shapes, 0)
    assert len(deep) == 1 and len(full) == 1, (deep, full)
    if n <= 64:
        assert "true" in deep[0] and "false" in full[0], (deep, full)
    else:
        assert "false" in deep[0] and "false" in full[0], (deep, full)


def test_hot_step_draws_the_same_masks():
    """The step forks the mask draws off the projection GEMM; they must still be the first two draws of torch's RNG after the
    seed, image first: the step with its own masks equals the step fed the two masks drawn directly."""
    import torch.nn.functional as F
    from tests.golden_util import Golden
    from mmssl_b200.engine import LIVE, FeatureStore
    from mmssl_b200.graph import prepare
    from mmssl_b200.hotstep import HotStep, HotStepConfig

    g = Golden("case_train_rand_k3")
    c = g.cfg
    cfg = HotStepConfig(embed_size=c["d"], n_layers=c["n_layers"], batch_size=c["B"])
    P = {k: v.clone().cuda().contiguous() for k, v in g.params.items()}
    hs = HotStep(P, (FeatureStore(g.image_feats.cuda()), FeatureStore(g.text_feats.cuda())),
                 [prepare(t) for t in g.graphs("cuda")], cfg, batch=len(g.users), optimizer_step=False)
    hs.set_indices(g.users, g.pos, g.neg)

    def step(masks):
        hs.masks = masks
        out = hs.run().clone()
        torch.cuda.synchronize()
        return out, {k: hs.grads[k].clone() for k in LIVE}

    torch.manual_seed(1234)
    out_a, grads_a = step(None)
    torch.manual_seed(1234)
    drawn = (F.dropout(hs.ones, cfg.drop_rate, True), F.dropout(hs.ones, cfg.drop_rate, True))
    out_b, grads_b = step(drawn)
    # the loss kernels add into their gradient seeds with float atomics, so the last bits may differ between two runs;
    # other masks would change the terms at the 1e-2 level
    assert torch.allclose(out_a, out_b, rtol=1e-6, atol=0), (out_a, out_b)
    for k in LIVE:
        scale = grads_b[k].abs().max().clamp_min(1e-30)
        assert float((grads_a[k] - grads_b[k]).abs().max() / scale) < 1e-5, k
