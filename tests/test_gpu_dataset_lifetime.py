"""ygg_dataset_destroy on a dataset that handles still use: the release waits for the last handle, which keeps training
on it meanwhile (the handle's destroy used to update the freed dataset's handle count)."""
import numpy as np
import pytest

import ydf_b200
from tests.util import synth

pytestmark = pytest.mark.gpu


def test_dataset_closed_before_its_handles():
    n = 20000
    bins, nb, na, y = synth(n, 6, seed=3, bins=64)
    ref_ds = ydf_b200.Dataset(bins, nb, na)
    ref = ydf_b200.Gbt(ref_ds, ydf_b200.default_config(max_depth=6, num_trees=3))
    ref.set_labels(y)
    ref.train(3)
    want = [ref.get_tree(i).tobytes() for i in range(3)]
    ref.close()
    ref_ds.close()

    ds = ydf_b200.Dataset(bins, nb, na)
    a = ydf_b200.Gbt(ds, ydf_b200.default_config(max_depth=6, num_trees=3))
    b = ydf_b200.Gbt(ds, ydf_b200.default_config(max_depth=6, num_trees=3))
    for g in (a, b):
        g.set_labels(y)
        g.train(1)
    ds.close()                     # both handles still use it
    a.train(2)
    assert [a.get_tree(i).tobytes() for i in range(3)] == want
    a.close()
    b.train(2)                     # the last handle: the dataset is still there
    assert [b.get_tree(i).tobytes() for i in range(3)] == want
    b.close()                      # releases the dataset
