"""Checkpoint file format (mmssl_b200/checkpoint.py) without kernels: the format tag, refusal of a checkpoint of another run
by field name, the atomic write, the training-matrix fingerprint, RNG states, and the Discriminator part under the
reference's keys."""
import os
import random
from types import SimpleNamespace

import numpy as np
import pytest
import scipy.sparse as sp
import torch

from mmssl_b200 import checkpoint


def _meta(**kw):
    cfg = SimpleNamespace(embed_size=64, n_layers=2, head_num=4)
    feats = (SimpleNamespace(dim=128), SimpleNamespace(dim=96))
    m = checkpoint.make_meta(100, 50, cfg, 1024, feats, (700, 12345))
    m.update(kw)
    return m


def _ckpt(**kw):
    return dict(format=checkpoint.FORMAT, kind="hotstep", meta=_meta(), model={"w": torch.arange(6.0).view(2, 3)}, **kw)


def test_format_tag_is_checked(tmp_path):
    p = str(tmp_path / "x.ckpt")
    torch.save(dict(format="something.else", model={}), p)
    with pytest.raises(ValueError, match="format"):
        checkpoint.load(p)
    torch.save({"model": {}}, p)
    with pytest.raises(ValueError, match="format"):
        checkpoint.load(p)
    with pytest.raises(ValueError, match="format"):
        checkpoint.save({"model": {}}, p)
    checkpoint.save(_ckpt(), p)
    assert checkpoint.load(p)["format"] == "mmssl_b200.ckpt.v1"
    with pytest.raises(ValueError, match="kind"):
        checkpoint.load(p, kinds=("trainer",))


@pytest.mark.parametrize("field,value", [("n_users", 101), ("n_items", 49), ("embed_size", 128), ("n_layers", 3), ("head_num", 2),
                                         ("batch_size", 2048), ("feat_widths", [128, 95]), ("train_nnz", 701),
                                         ("train_hash", 54321)])
def test_each_mismatched_field_is_refused_by_name(field, value):
    checkpoint.check_meta(_meta(), _meta())
    with pytest.raises(ValueError, match=field):
        checkpoint.check_meta(_meta(**{field: value}), _meta())


def test_tensor_shape_mismatch_is_refused_before_anything_is_copied():
    dst = {"a": torch.zeros(2, 3), "b": torch.zeros(4)}
    with pytest.raises(ValueError, match="model b"):
        checkpoint.copy_into(dst, {"a": torch.ones(2, 3), "b": torch.ones(5)}, "model")
    assert float(dst["a"].abs().sum()) == 0.0
    with pytest.raises(ValueError, match="'b'"):
        checkpoint.copy_into(dst, {"a": torch.ones(2, 3)}, "model")


def test_interrupted_write_leaves_the_previous_checkpoint(tmp_path, monkeypatch):
    p = str(tmp_path / "run.ckpt")
    checkpoint.save(_ckpt(), p)
    new = _ckpt()
    new["model"]["w"] = new["model"]["w"] + 100

    def fail(src, dst):
        raise OSError("simulated pre-emption before the rename")
    monkeypatch.setattr(os, "replace", fail)
    with pytest.raises(OSError):
        checkpoint.save(new, p)
    monkeypatch.undo()
    assert os.listdir(tmp_path) == ["run.ckpt"]                     # the partial temporary file is gone
    assert torch.equal(checkpoint.load(p)["model"]["w"], torch.arange(6.0).view(2, 3))
    checkpoint.save(new, p)
    assert torch.equal(checkpoint.load(p)["model"]["w"], new["model"]["w"])


def test_fingerprint_of_row_blocks_adds_up_and_tells_matrices_apart():
    rng = np.random.default_rng(0)
    R = sp.random(203, 131, density=0.05, format="csr", random_state=1)
    R.sort_indices()
    nnz, h = checkpoint.pattern_hash(R.indptr, R.indices, R.shape[1])
    assert nnz == R.nnz
    cut = 102
    a = checkpoint.pattern_hash(R.indptr[:cut + 1], R.indices, R.shape[1], row0=0)
    b = checkpoint.pattern_hash(R.indptr[cut:], R.indices, R.shape[1], row0=cut)
    assert a[0] + b[0] == nnz and (a[1] + b[1]) % (1 << 64) == h
    R2 = R.tolil()
    i, j = R.nonzero()
    R2[i[0], j[0]] = 0
    R2[i[0], (j[0] + 1 + int(rng.integers(0, 5))) % 131] = 1        # one edge moved
    R2 = R2.tocsr()
    R2.eliminate_zeros()
    R2.sort_indices()
    assert checkpoint.pattern_hash(R2.indptr, R2.indices, 131)[1] != h


def test_rng_states_round_trip_through_a_file(tmp_path):
    random.seed(3); np.random.seed(3); torch.manual_seed(3)
    random.random(); np.random.rand(5); torch.rand(5)
    p = str(tmp_path / "rng.ckpt")
    checkpoint.save(dict(format=checkpoint.FORMAT, kind="hotstep", rng=checkpoint.rng_state("cpu")), p)
    want = (random.random(), np.random.rand(3).tolist(), torch.rand(3))
    random.seed(9); np.random.seed(9); torch.manual_seed(9)
    checkpoint.set_rng_state(checkpoint.load(p)["rng"], "cpu")
    got = (random.random(), np.random.rand(3).tolist(), torch.rand(3))
    assert got[0] == want[0] and got[1] == want[1] and torch.equal(got[2], want[2])


def test_discriminator_part_loads_strict_into_the_reference_module(tmp_path):
    """gan.DiscriminatorState keeps the reference's state_dict keys; its Adam state sits beside it and loads in place."""
    import torch.nn as nn
    from mmssl_b200 import gan
    net = nn.Sequential(nn.Linear(64, 16), nn.LeakyReLU(True), nn.BatchNorm1d(16), nn.Dropout(0.3), nn.Linear(16, 8),
                        nn.LeakyReLU(True), nn.BatchNorm1d(8), nn.Dropout(0.5), nn.Linear(8, 1), nn.Sigmoid())
    D = gan.DiscriminatorState({"net." + k: v.detach().clone() for k, v in net.state_dict().items()})
    for k in gan.PARAMS:
        D.m[k].fill_(0.5)
        D.v[k].fill_(0.25)
    D.step = 7
    D.step_dev.fill_(7)
    p = str(tmp_path / "d.ckpt")
    checkpoint.save(dict(format=checkpoint.FORMAT, kind="fullstep", D=D.state_dict(), D_optim=D.optim_state_dict()), p)
    ck = checkpoint.load(p)

    class Discriminator(nn.Module):                  # the reference's module layout (Models.py:224-245)
        def __init__(self):
            super().__init__()
            self.net = net
    fresh = Discriminator()
    fresh.load_state_dict(ck["D"], strict=True)
    E = gan.DiscriminatorState({k: torch.zeros_like(v) for k, v in D.t.items()})
    E.load_state_dict(ck["D"], ck["D_optim"])
    assert E.step == 7 and int(E.step_dev[0]) == 7
    assert all(torch.equal(E.t[k], D.t[k]) for k in D.t) and all(torch.equal(E.m[k], D.m[k]) for k in gan.PARAMS)
    bad = dict(ck["D_optim"], step_dev=6)
    with pytest.raises(ValueError, match="D step"):
        E.load_state_dict(ck["D"], bad)


# ------------------------------------------------------------------------------------------ row-sharded checkpoints
def _rank_file(rank, world, step, U=5, I=3, d=4, **meta):
    """What RowShardedHotStep.state_dict() writes for `rank` of `world`, with entries that encode (step, global row)."""
    from mmssl_b200.engine import LIVE, P_EI, P_EU
    from mmssl_b200.parallel import RowPartition
    (ulo, uhi), (ilo, ihi) = RowPartition(U, world).bounds(rank), RowPartition(I, world).bounds(rank)
    rows = lambda lo, hi: (step * 1000 + torch.arange(lo, hi, dtype=torch.float32)).view(-1, 1).repeat(1, d)
    model = {P_EU: rows(ulo, uhi), P_EI: rows(ilo, ihi)}
    if rank == 0:
        model.update({k: torch.full((2, d), float(step)) for k in LIVE if k not in model})
    m = _meta(n_users=U, n_items=I, **meta)
    return dict(format=checkpoint.FORMAT, kind="rowshard", meta=m, rows={"user": (ulo, uhi), "item": (ilo, ihi)}, model=model,
                optim=dict(m={k: v + 0.5 for k, v in model.items()}, v={k: v + 0.25 for k, v in model.items()}, step=step))


def _write_generation(directory, world, step, ranks=None, commit=True, files=None):
    gen = f"step{step:010d}-world{world:05d}-a"
    os.makedirs(os.path.join(directory, gen), exist_ok=True)
    for r in (range(world) if ranks is None else ranks):
        f = files[r] if files is not None else _rank_file(r, world, step)
        checkpoint.save(f, checkpoint.shard_file(os.path.join(directory, gen), r, world))
    if commit:
        checkpoint.commit_sharded(directory, gen, world, step, _rank_file(0, world, step)["meta"])
    return gen


def test_sharded_files_of_different_saves_are_refused(tmp_path):
    d = str(tmp_path)
    # rank 1's file is still the one of step 3 next to rank 0's of step 5: never mixed into one state
    _write_generation(d, 2, 5, files={0: _rank_file(0, 2, 5), 1: _rank_file(1, 2, 3)})
    with pytest.raises(ValueError, match="step"):
        checkpoint.read_sharded(d, 1, 0)
    d2 = str(tmp_path / "other_run")
    _write_generation(d2, 2, 5, files={0: _rank_file(0, 2, 5), 1: _rank_file(1, 2, 5, train_hash=999)})
    with pytest.raises(ValueError, match="meta"):
        checkpoint.read_sharded(d2, 1, 0)
    with pytest.raises(ValueError, match="MANIFEST"):
        checkpoint.read_sharded(str(tmp_path / "nothing"), 1, 0)


def test_sharded_save_commits_whole_generations_only(tmp_path):
    from mmssl_b200.engine import P_EU
    d = str(tmp_path)
    one_rank = lambda st: SimpleNamespace(state_dict=lambda: st, pu=SimpleNamespace(world=1), rank=0, group=None)
    checkpoint.save_sharded(one_rank(_rank_file(0, 1, 3)), d)
    assert checkpoint.read_sharded(d, 2, 1)["optim"]["step"] == 3
    # a save at world 2 pre-empted after rank 0's file: the committed checkpoint is still the whole one of step 3
    _write_generation(d, 2, 7, ranks=[0], commit=False)
    full = checkpoint.read_sharded(d, 1, 0)
    assert full["optim"]["step"] == 3 and torch.equal(full["model"][P_EU][:, 0], 3000 + torch.arange(5.0))
    # the complete world-2 save replaces it; the files of other world sizes and saves are removed
    gen = _write_generation(d, 2, 7)
    assert sorted(os.listdir(d)) == sorted([checkpoint.MANIFEST, gen])
    blk = checkpoint.read_sharded(d, 2, 1)                       # rows 3, 4 of 5 and zero padding, from the two files
    assert blk["optim"]["step"] == 7 and blk["model"][P_EU][:, 0].tolist() == [7003.0, 7004.0, 0.0]
    # saving the same step again never rewrites the committed files in place
    checkpoint.save_sharded(one_rank(_rank_file(0, 1, 7)), d)
    assert sorted(os.listdir(d)) == [checkpoint.MANIFEST, "step0000000007-world00001-a"]
    checkpoint.save_sharded(one_rank(_rank_file(0, 1, 7)), d)
    assert sorted(os.listdir(d)) == [checkpoint.MANIFEST, "step0000000007-world00001-b"]
    assert checkpoint.read_sharded(d, 1, 0)["optim"]["step"] == 7


def test_device_sampler_seed_is_compared_when_both_runs_have_one():
    checkpoint.check_meta(_meta(), _meta(sampler_seed=4))
    checkpoint.check_meta(_meta(sampler_seed=4), _meta(sampler_seed=4))
    with pytest.raises(ValueError, match="sampler_seed"):
        checkpoint.check_meta(_meta(sampler_seed=4), _meta(sampler_seed=5))
