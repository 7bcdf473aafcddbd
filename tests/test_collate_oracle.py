"""CPU: the packed-collation oracle (oracle/collate_oracle.py) against what the unmodified reference makes of the same batch
(tests/golden/collate.pt from tests/golden/make_golden_collate.py): `_featurize_as_graph` + collation + `prepare_context`,
restricted to mask == True rows — bit-exact."""
import os

import numpy as np
import pytest
import torch

import collate_layouts as CL
import collate_oracle as CO
from conftest import GOLDEN


def test_packed_batch_equals_reference_batch_restricted_to_mask():
    fx = torch.load(os.path.join(GOLDEN, "collate.pt"), weights_only=False)
    x, oh, ch, bi, counts = CO.collate_packed(fx["positions"].numpy(), fx["charges"].numpy(), fx["one_hot"].numpy(),
                                              fx["idx"].numpy())
    ref = fx["ref"]
    assert np.array_equal(x, ref["x"].numpy()) and np.array_equal(oh, ref["one_hot"].numpy())
    assert np.array_equal(ch, ref["charges"].numpy()) and np.array_equal(bi, ref["batch"].numpy())
    assert counts.sum() == ref["present_rows"] < ref["padded_rows"]
    ctx = CO.prepare_context([fx["alpha"].numpy(), fx["mu"].numpy()], fx["idx"].numpy(), bi,
                             [fx["norms"]["alpha"]["mean"].item(), fx["norms"]["mu"]["mean"].item()],
                             [fx["norms"]["alpha"]["mad"].item(), fx["norms"]["mu"]["mad"].item()])
    assert np.array_equal(ctx, ref["context"].numpy())


@pytest.mark.parametrize("kind", list(CL.BATCHES))
@pytest.mark.parametrize("num_types", CL.NUM_TYPES)
@pytest.mark.parametrize("pad", CL.PADS)
def test_torch_reference_of_synthetic_layouts_equals_oracle(pad, num_types, kind):
    """The plain torch expression tests/test_gpu_collate_layouts.py compares the kernels with, on every synthetic layout
    (pads 29 .. 200, 5 and 16 types, holes, empty molecules, repeated and unsorted ids, 1 to 3 properties), against the
    oracle pinned to the reference: bit-exact."""
    data, norms = CL.padded_dataset(pad, num_types)
    idx = CL.batch_ids(kind, data["charges"].shape[0])
    cond = CL.BATCHES[kind]
    ref = CL.packed_reference(data, norms, idx, cond)
    x, oh, ch, bi, counts = CO.collate_packed(data["positions"].numpy(), data["charges"].numpy(), data["one_hot"].numpy(),
                                              idx.numpy())
    assert np.array_equal(x, ref["x"].numpy()) and np.array_equal(oh, ref["one_hot"].numpy())
    assert np.array_equal(ch, ref["charges"].numpy()) and np.array_equal(bi, ref["batch"].numpy())
    assert np.array_equal(counts, ref["counts"].numpy())
    ctx = CO.prepare_context([data[k].numpy() for k in cond], idx.numpy(), bi, [norms[k]["mean"].item() for k in cond],
                             [norms[k]["mad"].item() for k in cond])
    assert np.array_equal(ctx, ref["context"].numpy())
    if kind != "one":                                        # the batch reaches the layouts it is meant to
        assert (counts == 0).any() and (ref["charges"] > 0).all() and (data["charges"][idx] < 0).any()
