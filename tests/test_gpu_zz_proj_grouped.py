"""The grouped, persistent projection GEMM (csrc/proj_tc.cu, gemm_bf16x3_group_kernel) on the H100: image and text of one
direction in one launch.  Checked against fp64 products through the existing split-K epilogues, and bitwise against the
single-problem kernel's partials when both use the same slices.  tests/test_emu_proj_grouped.py runs the same bodies at
small sizes in the emulator."""
import pytest
import torch

from tests.golden_util import rel_err

pytestmark = pytest.mark.gpu

K_MAX_CHAIN_KB = 48   # csrc/tc_common.cuh kMaxChainKb


def _operands(m, n, k, seed):
    from mmssl_b200 import ops
    g = torch.Generator().manual_seed(seed)
    a = torch.randn(m, k, generator=g).cuda()
    b = (torch.randn(n, k, generator=g) * 0.05).cuda()
    return a, b, ops.split_bf16(a), ops.split_bf16(b)


def _run_group(shapes, max_ctas=0, splits=None, seed=11):
    """shapes: [(m, n, k), ...].  Returns [(a, b, split, partial)] after one grouped launch."""
    from mmssl_b200 import ops
    plan_splits, _ = ops.gemm_bf16x3_group_plan(shapes, max_ctas)
    splits = plan_splits if splits is None else splits
    out, probs = [], []
    for p, ((m, n, k), sk) in enumerate(zip(shapes, splits)):
        a, b, (a_hi, a_lo), (b_hi, b_lo) = _operands(m, n, k, seed + p)
        part = torch.full((sk * m * n,), float("nan"), device="cuda")
        probs.append((a_hi, a_lo, b_hi, b_lo, m, n, k, sk, part))
        out.append((a, b, sk, part))
    ops.gemm_bf16x3_group(probs, max_ctas)
    torch.cuda.synchronize()
    return out


def check_group_vs_fp64(shapes, max_ctas=0):
    """Forward (proj_epilogue: bias + mask) and weight-gradient (wgrad_epilogue) reductions of every problem's partials
    against the fp64 product, at the tolerance of the single-problem test (test_gpu_ops.test_gemm_bf16x3_tensor_core)."""
    from mmssl_b200 import ops
    for p, (a, b, sk, part) in enumerate(_run_group(shapes, max_ctas)):
        m, n, _ = shapes[p]
        want = a.double().cpu() @ b.double().cpu().t()
        bias = torch.randn(n).cuda()
        mask = ((torch.rand(m, n) > 0.2).float() / 0.8).cuda()
        y = torch.empty(m, n, device="cuda")
        y_pre = torch.empty(m, n, device="cuda")
        ops.proj_epilogue(part, sk, m, n, bias, mask, y, y_pre)
        assert rel_err(y_pre, want + bias.double().cpu()) < 2e-5
        assert rel_err(y, (want + bias.double().cpu()) * mask.double().cpu()) < 2e-5
        dw = torch.empty(n, m, device="cuda")
        ops.wgrad_epilogue(part, sk, m, n, dw)
        assert rel_err(dw, want.t()) < 2e-5


def check_group_bitwise_vs_single(shapes, max_ctas=0):
    """With each problem's single-kernel plan, the grouped launch writes exactly the partials mmssl_gemm_bf16x3 writes."""
    from mmssl_b200 import ops
    splits = [ops.gemm_bf16x3_plan(*s)[1] for s in shapes]
    got = _run_group(shapes, max_ctas, splits=splits)
    for p, (m, n, k) in enumerate(shapes):
        _, _, (a_hi, a_lo), (b_hi, b_lo) = _operands(m, n, k, 11 + p)
        ref = torch.full((splits[p] * m * n,), float("nan"), device="cuda")
        ops.gemm_bf16x3(a_hi, a_lo, b_hi, b_lo, m, n, k, splits[p], ref)
        assert torch.equal(got[p][3].cpu(), ref.cpu()), f"problem {p}: grouped partials differ from the single kernel's"


def check_plan(shapes, max_ctas=0):
    """The unit list covers every (problem, m_tile, k-block) exactly once, in slices of the planned split, no unit longer
    than kMaxChainKb k-blocks, longest first."""
    from mmssl_b200 import ops
    splits, floats, units = ops.gemm_bf16x3_group_plan(shapes, max_ctas, units=True)
    u = units.numpy()
    assert (u[:, 3] - u[:, 2] <= K_MAX_CHAIN_KB).all() and (u[:, 3] > u[:, 2]).all()
    lens = u[:, 3] - u[:, 2]
    assert (lens[:-1] >= lens[1:]).all(), "units are not sorted longest first"
    for p, (m, n, k) in enumerate(shapes):
        assert floats[p] == splits[p] * m * n
        mt, kb = (m + 127) // 128, (k + 63) // 64
        cover = torch.zeros(mt, kb, dtype=torch.int32)
        sel = u[u[:, 0] == p]
        assert len(sel) == splits[p] * mt
        for _, t, k0, k1 in sel:
            cover[t, k0:k1] += 1
        assert bool((cover == 1).all())
    return splits


BABY_FWD = [(7050, 64, 4096), (7050, 64, 1024)]
BABY_WGRAD = [(4096, 64, 7050), (1024, 64, 7050)]
SPORTS_FWD = [(18357, 64, 4096), (18357, 64, 1024)]
SPORTS_WGRAD = [(4096, 64, 18357), (1024, 64, 18357)]


@pytest.mark.parametrize("shapes", [BABY_FWD, BABY_WGRAD, SPORTS_FWD, SPORTS_WGRAD], ids=["baby_fwd", "baby_wgrad", "sports_fwd", "sports_wgrad"])
def test_group_vs_fp64(shapes):
    check_group_vs_fp64(shapes)


@pytest.mark.parametrize("shapes", [BABY_FWD, SPORTS_FWD, BABY_WGRAD], ids=["baby_fwd", "sports_fwd", "baby_wgrad"])
def test_group_bitwise_vs_single_kernel(shapes):
    check_group_bitwise_vs_single(shapes)


def test_group_n128_and_one_problem():
    check_group_vs_fp64([(5000, 128, 4096), (5000, 128, 1024)])
    check_group_vs_fp64([(7050, 64, 4096)])


@pytest.mark.parametrize("shapes", [BABY_FWD, BABY_WGRAD, SPORTS_FWD, SPORTS_WGRAD], ids=["baby_fwd", "baby_wgrad", "sports_fwd", "sports_wgrad"])
def test_group_plan(shapes):
    check_plan(shapes)


def test_baby_forward_keeps_the_single_kernel_slices():
    from mmssl_b200 import ops
    assert check_plan(BABY_FWD) == [ops.gemm_bf16x3_plan(*s)[1] for s in BABY_FWD]
