"""The oracle restatement against the UNMODIFIED reference classes on freshly seeded parity cases.  The reference's
indices, prediction, loss and table gradients were recorded once by oracle/make_golden.py (make_live_cases, with
oracle/kaolin_shim) into tests/golden/ref_live_cases.npz; the cases are rebuilt here from their seeds."""
import os

import numpy as np
import pytest

from tests.parity_utils import ROOT, make_case, run_oracle_step

GOLDEN = os.path.join(ROOT, "tests", "golden", "ref_live_cases.npz")


@pytest.mark.parametrize("levels,frames,poly", [(2, 1, True), (4, 2, True), (3, 2, False)])
def test_oracle_equals_live_reference(levels, frames, poly):
    ref = np.load(GOLDEN)
    key = f"l{levels}_f{frames}_p{int(poly)}_"
    case = make_case(n_points=1200, n_batch=1000, feat_levels=levels, seed=77 + levels, n_frames=frames, poly=poly)
    assert np.array_equal(case["coord"], ref[key + "coord"]), "the seeded case no longer matches the recorded one"
    want = run_oracle_step(case)
    for i, b in enumerate(want["indices"]):
        assert np.array_equal(ref[key + f"indices_{i}"], b)
    assert np.abs(ref[key + "pred"] - want["pred"]).max() < 1e-6
    assert abs(float(ref[key + "loss"]) - want["loss"]) < 1e-6
    for i, g in enumerate(want["table_grads"]):
        assert np.abs(ref[key + f"tgrad_{i}"] - g).max() <= 1e-5 * np.abs(g).max() + 1e-12
