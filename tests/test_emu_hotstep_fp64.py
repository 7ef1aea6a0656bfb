"""tests/test_gpu_zz_hotstep_fp64.py executed on the CPU by the cuemu fiber emulator (tests/cuemu) at small sizes: the hot step
against float64 per loss term, per class of rows (the SpMM plan's cuts lowered so that a 200-row graph has split and heavy
rows), on awkward batches, over optimiser steps that change batch and masks, and the AdamW update.  Full-size and
captured-graph cases run on the GPU only; the wgmma projection is the emulator's host statement of its contract."""
import pytest

from tests import test_gpu_zz_hotstep_fp64 as G
from tests.cuemu import harness

CUTS = (8, 4, 32, 8)
SMALL = dict(U=203, I=157, B=48, cuts=CUTS)


@pytest.fixture(params=["fwd", "rev"])
def emu(request, monkeypatch):
    harness.set_order(request.param)
    return harness.emulated_device(monkeypatch)


@pytest.fixture
def emu_fwd(monkeypatch):
    harness.set_order("fwd")
    return harness.emulated_device(monkeypatch)


@pytest.fixture
def cuts(emu_fwd):
    from mmssl_b200 import ops
    ops.spmm_plan_set_cuts(*CUTS)
    yield ops.spmm_plan_set_cuts
    ops.spmm_plan_set_cuts(*G.H.DEFAULT_CUTS)


@pytest.mark.parametrize("term", G.TERMS)
def test_each_loss_term(cuts, term):
    G.check_terms(term, "simt/simt", **SMALL)


@pytest.mark.parametrize("term", ["default", "emb_reg dominant", "infonce dominant"])
def test_each_loss_term_tensor_cores(cuts, term):
    G.check_terms(term, "tc/auto", modal="alias", **SMALL)


@pytest.mark.parametrize("d,K,head_num,modal,route", [
    (64, 2, 4, "distinct", "simt/simt"), (64, 3, 1, "alias", "tc/auto"), (128, 1, 4, "empty", "simt/auto"),
    (32, 4, 1, "distinct", "tc/simt"), (96, 2, 4, "alias", "simt/simt"), (192, 1, 1, "distinct", "simt/simt"),
    (256, 2, 4, "alias", "tc/simt")])
def test_row_classes(emu, d, K, head_num, modal, route):
    from mmssl_b200 import ops
    try:
        G.check_row_classes(d, K, head_num, modal, route, U=203, I=157, B=48, dv=24, dt=20, cuts=CUTS, set_cuts=ops.spmm_plan_set_cuts)
    finally:
        ops.spmm_plan_set_cuts(*G.H.DEFAULT_CUTS)


@pytest.mark.parametrize("route", ["simt/simt", "tc/auto"])
@pytest.mark.parametrize("kind", G.AWKWARD)
def test_awkward_batches(cuts, kind, route):
    G.check_awkward(kind, route, **SMALL)


@pytest.mark.parametrize("B", [1, 2, 63, 65, 257])
def test_batch_sizes(cuts, B):
    G.check_batch_size(B, "simt/auto", U=203, I=157, cuts=CUTS)


@pytest.mark.parametrize("modal,route,mode", [("distinct", "simt/simt", "eager"), ("empty", "simt/simt", "eager"),
                                              ("alias", "tc/auto", "eager")])
def test_steps_from_device_state(cuts, modal, route, mode):
    G.check_replays(modal, route, mode, n=4, **SMALL)


@pytest.mark.parametrize("step,wd,lr", [(1, 1e-2, 5.5e-4), (2, 1.0, 5.5e-4), (10, 0.0, 1e-1), (1000, 1e-2, 1e-1), (100000, 1.0, 5.5e-4)])
def test_adamw_update_in_step(emu_fwd, step, wd, lr):
    G.check_adamw_in_step(step, wd, lr)


@pytest.mark.parametrize("gan", [False, True])
def test_adamw_many_tensors(emu, gan):
    G.check_adamw_many_tensors(gan)


def test_adamw_zero_gradient_is_exactly_the_decay(emu):
    G.check_adamw_zero_gradient()
