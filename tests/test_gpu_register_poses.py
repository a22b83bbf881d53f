"""shine_register_normal_eq_poses on the GPU: every row equals the single-pose entry bit for bit, and a short scratch
is refused."""
import ctypes as C

import numpy as np
import pytest
import torch

from shine_mapping_b200 import _abi
from tests.test_gpu_odometry import _random_pose, _scan, _trained

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


# ---- the K-pose entry against the single-pose entry ------------------------------------------------------------------------

@pytest.fixture(scope="module")
def trained():
    return _trained(0)


def _poses(rng, K, scale):
    """K poses around the scan's own; every seventh far off the map (every point masked)."""
    P = np.stack([_random_pose(rng, scale) for _ in range(K)])
    P[3::7, :3, 3] = (3.0, -3.0, 3.0)
    return P


@pytest.mark.parametrize("n", [0, 1, 256 * 3 + 37, 10 ** 6])
@pytest.mark.parametrize("K", [1, 2, 1105, "split"])
def test_poses_entry_equals_the_single_pose_entry_bit_for_bit(trained, n, K):
    """Row k of launch_poses is launch at pose k, bit for bit.  "split": 1300 poses with a scratch bound of 700 poses,
    so launch_poses makes two calls and the entry launches its 512-pose chunks within each."""
    case, reg = trained
    rng = np.random.default_rng(100 + n)
    world = _scan(case, rng, max(n, 1), 0.05, reg.scale).astype(np.float32)
    pts = torch.from_numpy(world[:n].reshape(-1, 3)).to(DEV)
    split = K == "split"
    K = 1300 if split else K
    P = _poses(rng, K, reg.scale)
    kappa = 0.1 * reg.scale
    want = torch.full((K, _abi.REGISTER_OUT), float("nan"), dtype=torch.float64, device=DEV)
    for k in range(K):
        reg.launch(pts, P[k], kappa, want[k])
    got = torch.full_like(want, float("nan"))
    if split:
        reg.SCRATCH_BOUND_BYTES = 700 * _abi.lib().shine_register_scratch_bytes(n, 1)
    try:
        reg.launch_poses(pts, P, kappa, got)
    finally:
        reg.__dict__.pop("SCRATCH_BOUND_BYTES", None)
    got, want = got.cpu().numpy(), want.cpu().numpy()
    assert np.array_equal(got.view(np.int64), want.view(np.int64)), np.argwhere(got != want)[:5]
    off = got[3::7]
    assert np.array_equal(off, np.zeros_like(off)), "poses off the map have no valid point"
    if n >= 256:
        assert (got[:, 28] > 0).sum() >= K // 2, "most poses put points on the map"


def test_poses_entry_refuses_a_short_scratch_on_the_device(trained):
    case, reg = trained
    pts = torch.zeros(5000, 3, device=DEV)
    lib = _abi.lib()
    need = lib.shine_register_scratch_bytes(5000, 3)
    assert need == 20 * 3 * 29 * 8
    scratch = torch.empty(need, dtype=torch.uint8, device=DEV)
    out = torch.empty(3, 29, dtype=torch.float64, device=DEV)
    od, dd = reg.octree._descriptor(None, None), reg.decoder.c_descriptor(None)
    poses = (C.c_double * 48)(*np.tile(np.eye(4).reshape(-1), 3).tolist())
    call = lambda sb: lib.shine_register_normal_eq_poses(C.byref(od), C.byref(dd), _abi.ptr(pts), 5000, poses, 3,
                                                         reg.sigma, 0.1, _abi.ptr(out), _abi.ptr(scratch), sb, None)
    assert call(need - 8) == -1
    assert call(need) == 0
    torch.cuda.synchronize()
