"""The tensor-core neighbour pass parks each epilogue warp's candidates (superposed) or edges (unsuperposed) in shared
memory and flushes them to the global list in batches. Identical fingerprints make every pair of the tile a hit, so each
warp fills and flushes its slots many times per tile; the list must hold each hit exactly once."""

import numpy as np
import pytest
import torch

from nvmolkit_b200 import synthetic as S

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("cluster", [0, 1, 3])
@pytest.mark.parametrize("rows,cols", [(4, 4), (2, 1), (1, 1)])
def test_every_hit_of_a_dense_tile_is_listed_once(cuda, cluster, rows, cols):
    from nvmolkit_b200 import _lib
    from nvmolkit_b200.clustering import fused_butina_device

    n = 2000  # a multiple of every superposition factor: no partial super row or column
    one = np.repeat(S.random_fingerprints(1, bits=1024, seed=11), n, axis=0)
    with _lib.options(similarity_tensor_min_pairs=0, similarity_tensor_cluster=cluster, similarity_superpose=rows,
                      similarity_superpose_cols=cols):
        ids, cen = fused_butina_device(torch.from_numpy(one.view(np.int32)).to(cuda), 0.3)
        assert _lib.get_option("similarity_superpose_last") == rows * cols
        listed = _lib.get_option("similarity_candidates_last")
    assert (ids.cpu().numpy() == 0).all() and cen.cpu().numpy().tolist() == [n - 1]
    if rows * cols > 1:
        # candidate (super row R, super column J) <=> the group holds a pair i < j: R rows < (J + 1) cols - 1
        R = np.arange(n // rows)[:, None]
        J = np.arange(n // cols)[None, :]
        assert listed == int((R * rows < (J + 1) * cols - 1).sum())
