"""FactorGraph.update / update_lowmem: the restatement oracle.factor_graph against the state the UNMODIFIED reference methods left on the
same stub graph and CPU operators (tests/golden/make_factor_graph_golden.py); bit-exact.  Where the reference tree is present the
methods are re-run live.  Also the properties of the update_lowmem hook's chunk planner (droid_slam_b200.modules.plan_lowmem_chunks)."""
import os
import sys

import pytest
import torch

import oracle.factor_graph as ofg
from droid_slam_b200.modules import plan_lowmem_chunks

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
import make_factor_graph_golden as mk  # noqa: E402

REF_PRESENT = os.path.isdir(os.path.join(mk.REF, "droid_slam"))
CASES = {c[0]: c for c in mk.cases()}


@pytest.fixture(scope="module")
def gold():
    return torch.load(os.path.join(ROOT, "tests", "golden", "factor_graph.pt"))


def run_oracle(case):
    graph, kw = mk.make(case)
    if case[1] == "update":
        ofg.update(graph, **kw)
    else:
        ofg.update_lowmem(graph, alt_corr_block=mk.AltCorrBlock, **kw)
    return mk.stored(mk.state(graph))


def _assert_state_equal(got, gold, name):
    for k, t in got.items():
        assert torch.equal(t, gold[name + "/" + k]), (name, k)


@pytest.mark.parametrize("name", list(CASES))
def test_restatement_matches_the_reference_methods(gold, name):
    _assert_state_equal(run_oracle(CASES[name]), gold, name)


def test_cases_exercise_the_reference_behaviours(gold):
    # the quirk case leaves the edges beyond the reference's last chunk untouched but still runs BA on them
    graph, _ = mk.make(CASES["lowmem_quirk"])
    uncovered = graph.ii >= 8
    assert ofg.lowmem_chunk_starts(graph.ii, graph.jj) == [0] and bool(uncovered.any())
    assert torch.equal(gold["lowmem_quirk/target"][:, uncovered], graph.target[:, uncovered])
    assert torch.equal(gold["lowmem_quirk/weight"][:, uncovered], graph.weight[:, uncovered])
    assert not torch.equal(gold["lowmem_quirk/target"][:, ~uncovered], graph.target[:, ~uncovered])
    assert not torch.equal(gold["lowmem_quirk/poses"][8:], graph.video.poses[8:])
    # update_lowmem marks every frame dirty, update does not; upsampling wrote disps_up
    assert bool(gold["lowmem_rig1_inac/dirty"].all()) and not bool(gold["update_inac_t0none/dirty"].any())
    assert not torch.equal(gold["update_inac_t0none/disps_up"], mk.digest(torch.zeros(9, 8 * mk.HT, 8 * mk.WD)))
    # motion_only BA keeps the depths
    graph, _ = mk.make(CASES["update_motion_only"])
    assert torch.equal(gold["update_motion_only/disps"], graph.video.disps.clamp(min=0.001))


@pytest.mark.skipif(not REF_PRESENT, reason="reference tree not present")
def test_reference_methods_reproduce_the_fixture(gold):
    fg = mk.import_reference_factor_graph()
    for name, case in CASES.items():
        _assert_state_equal(mk.run_reference(fg, case), gold, name)


def _reference_coverage(ii, jj):
    """edges the reference's update_lowmem loop passes to the update operator, each chunk's edges in graph order"""
    out = []
    for first in range(int(ii.min()), int(jj.max()) + 1, 8):
        sel = torch.nonzero((ii >= first) & (ii < first + 8))[:, 0]
        if sel.numel():
            out.append(sel)
    return torch.cat(out) if out else torch.zeros(0, dtype=torch.long)


@pytest.mark.parametrize("seed,n_frames,n_edges,budget", [(0, 40, 300, 30), (1, 40, 300, 7), (2, 12, 60, 1000), (3, 90, 900, 64),
                                                           (4, 30, 200, 1)])
def test_lowmem_plan_properties(seed, n_frames, n_edges, budget):
    g = torch.Generator().manual_seed(seed)
    ii = torch.randint(0, n_frames, (n_edges,), generator=g)
    jj = (ii + torch.randint(-5, 6, (n_edges,), generator=g)).clamp(0, n_frames - 1)
    if seed == 3:                                    # sources far beyond jj.max(): the chunk coverage quirk
        jj = jj.clamp(max=n_frames // 2)
    perm, chunks, src, seg = plan_lowmem_chunks(ii, jj, budget)
    covered = _reference_coverage(ii, jj)
    # every covered edge exactly once, nothing else
    assert torch.equal(torch.sort(perm).values, torch.sort(covered).values)
    if seed == 3:
        assert perm.numel() < n_edges
    assert chunks[0][0] == 0 and chunks[-1][1] == perm.numel() and chunks[-1][3] == src.numel()
    seen = set()
    for (a, b, s0, s1), nxt in zip(chunks, chunks[1:] + [None]):
        if nxt is not None:
            assert nxt[0] == b and nxt[2] == s1
        rows = perm[a:b]
        frames = ii[rows]
        # graph order inside a chunk, whole source frames, ascending frame list and segment ranks like torch.unique
        assert bool((rows[1:] > rows[:-1]).all())
        uniq, inv = torch.unique(frames, return_inverse=True)
        assert torch.equal(src[s0:s1], uniq) and torch.equal(seg[a:b], inv)
        assert not (set(uniq.tolist()) & seen)
        seen |= set(uniq.tolist())
        # the budget holds unless the chunk is one oversized source frame
        assert b - a <= budget or uniq.numel() == 1
    assert seen == set(ii[covered].tolist())


def test_lowmem_plan_nothing_covered():
    # every source frame lies beyond jj.max(): range(ii.min(), jj.max() + 1, 8) is empty and the reference updates no edge
    perm, chunks, src, seg = plan_lowmem_chunks(torch.tensor([9, 10, 12]), torch.tensor([2, 3, 1]), 100)
    assert perm.numel() == 0 and chunks == [] and src.numel() == 0
