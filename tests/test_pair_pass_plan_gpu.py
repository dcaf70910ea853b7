"""The sequence of tensor-core passes a neighbour-pass call plans: the superposition factor it reports and the units it
sized its grids for, summed over every pass of the call (similarity_units_planned_last), after a whole-call overflow,
after pipeline chunks that overflow at 4 x 4 and at 4 x 1, and at a factor the pilot chose. The expected units are
tools/pilot_model.group_units over the popcount band of each pass (band_ends); clusters and centroids must equal those
of the unsuperposed pass.

Where a superposed list overflows, every live (super row, super column) pair of these sets is a candidate: identical
fingerprints, or half-dense random ones, whose 4 summed intersections (about 2,000) lie far above the pre-filter's bar
(about 0.41 x 2 x 1,024)."""

import numpy as np
import pytest
import torch

import test_path_a_gpu as A
from nvmolkit_b200 import synthetic as S
from tools import pilot_model as M

pytestmark = pytest.mark.gpu

CUTOFF = 0.3


def _units(fp, s, c):
    """Units of one symmetric pass over all row groups at s x c (CTA pairs), within the popcount band; a pass over a
    subset of the row groups plans the units of those groups, so passes that split the groups between them sum to this."""
    pop = np.sort(M.popcounts(fp))
    ends = M.band_ends(pop, pop, M.thresh_table(32 * fp.shape[1], CUTOFF), M.TILE_N * c)
    return int(M.group_units(len(fp), s, c, ends, pair=True, run=1).sum())


def _run(fp, cuda, **opts):
    """Fused Butina at the given options, then unsuperposed: (superpose_last, units_planned_last); asserts that both
    passes give the same clusters."""
    from nvmolkit_b200 import _lib
    from nvmolkit_b200.clustering import fused_butina_device

    dev = A._dev(fp, cuda)
    with _lib.options(similarity_tensor_min_pairs=0, similarity_tensor_cluster=1, similarity_popcount_band=1, **opts):
        ids, cen = fused_butina_device(dev, CUTOFF)
        got = _lib.get_option("similarity_superpose_last"), _lib.get_option("similarity_units_planned_last")
        with _lib.options(similarity_superpose=1, similarity_superpose_cols=1):
            ids1, cen1 = fused_butina_device(dev, CUTOFF)
    assert torch.equal(ids, ids1) and torch.equal(cen, cen1)
    return got


def _dense_clusters(centres, members, seed):
    """Half-dense random 2048-bit centres, each repeated `members` times: neighbours only within a centre's copies."""
    rng = np.random.default_rng(seed)
    fp = np.repeat(S.pack_bits(rng.random((centres, 2048)) < 0.5), members, axis=0)
    return np.ascontiguousarray(fp[rng.permutation(len(fp))])


def test_whole_call_overflow_steps_down_to_rows_then_to_single_pairs(cuda):
    """12,000 identical fingerprints (two row groups, no pipeline): 4 x 4 and 4 x 1 overflow, 1 x 1 completes."""
    fp = np.repeat(S.random_fingerprints(1, seed=3), 12000, axis=0)
    last, planned = _run(fp, cuda, similarity_superpose=4, similarity_superpose_cols=4, similarity_superpose_auto=0)
    assert last == 1
    assert planned == _units(fp, 4, 4) + _units(fp, 4, 1) + _units(fp, 1, 1)


def test_pipeline_chunks_that_overflow_at_4x4_are_redone_from_4x1(cuda):
    """17 row groups: 4 chunks at 4 x 4, each overflows its quarter of the list; each is redone on its own at 4 x 1 with
    the whole list, overflows again and completes at 1 x 1. The call still reports 4 x 4."""
    fp = _dense_clusters(13108, 10, seed=1)
    last, planned = _run(fp, cuda, similarity_superpose=4, similarity_superpose_cols=4, similarity_superpose_auto=0,
                         similarity_pipeline_chunks=4)
    assert last == 16
    assert planned == _units(fp, 4, 4) + _units(fp, 4, 1) + _units(fp, 1, 1)


def test_pipeline_chunks_that_overflow_at_4x1_are_redone_at_4x1(cuda):
    """The same at 4 x 1: a chunk that overflows its quarter of the list reruns 4 x 1 with the whole list first."""
    fp = _dense_clusters(13108, 10, seed=2)
    last, planned = _run(fp, cuda, similarity_superpose=4, similarity_superpose_cols=1, similarity_superpose_auto=0,
                         similarity_pipeline_chunks=4)
    assert last == 4
    assert planned == 2 * _units(fp, 4, 1) + _units(fp, 1, 1)


def test_pilot_chosen_factor_plans_one_pass(cuda):
    """70,000 dense fingerprints: the pilot picks a narrower factor than 4 x 4 (test_pair_pass_popcount_order_gpu pins
    the choice to the CPU model); its passes are not counted, the call plans the one pass at the chosen factor."""
    fp = S.random_fingerprints(70_000, p=0.08, seed=5, near_dups=30_000)
    last, planned = _run(fp, cuda, similarity_superpose=4, similarity_superpose_cols=4, similarity_superpose_auto=1,
                         similarity_pipeline_chunks=4)
    assert last in (4, 8)
    assert planned == _units(fp, 4, last // 4)
