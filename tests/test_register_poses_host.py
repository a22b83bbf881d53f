"""Host side of the K-pose normal equations: the argument checks of shine_register_normal_eq_poses and its scratch size,
and the batches launch_poses makes."""
import ctypes as C
import numpy as np
import pytest
import torch

from shine_mapping_b200 import odometry


def test_poses_entry_argument_checks_need_no_gpu(built_lib):
    from shine_mapping_b200 import _abi
    lib = built_lib
    slots = (C.c_uint8 * 64)()
    feats = (C.c_float * 8)()
    oct_ = _abi.ShineOctree()
    oct_.num_levels, oct_.feature_dim = 1, 8
    lv = oct_.lv[0]
    lv.hash_slots, lv.features, lv.hash_capacity, lv.rows, lv.level = C.addressof(slots), C.addressof(feats), 1, 1, 12
    w = (C.c_float * 1024)()
    dec = _abi.ShineDecoder()
    dec.w1 = dec.w2 = dec.w3 = C.addressof(w)
    dec.in_dim, dec.hidden, dec.mlp_level = 8, 32, 2
    K = 3
    poses = (C.c_double * (16 * K))(*np.tile(np.eye(4).reshape(-1), K).tolist())
    out = (C.c_double * (29 * K))()
    scratch = C.addressof((C.c_double * 8)())
    pts = C.addressof((C.c_float * 3)())
    need = lib.shine_register_scratch_bytes(1, K)
    assert need == K * 29 * 8

    def call(o=oct_, d=dec, points=pts, n=1, p=poses, k=K, sigma=1.0, kappa=0.1, o_ut=out, s=scratch, sb=need):
        return lib.shine_register_normal_eq_poses(C.byref(o) if o is not None else None,
                                                  C.byref(d) if d is not None else None, points, n, p, k, sigma, kappa,
                                                  C.addressof(o_ut) if o_ut is not None else None, s, sb, None)

    assert call(k=0) == -1 and call(k=-2) == -1 and call(k=2 ** 31) == -1
    assert call(p=None) == -1 and call(o_ut=None) == -1
    assert call(o=None) == -1 and call(d=None) == -1 and call(points=None) == -1 and call(n=-1) == -1
    assert call(s=None) == -1 and call(sb=need - 8) == -1 and call(s=scratch + 4) == -1
    for bad in (0.0, -1.0, float("nan"), float("inf")):
        assert call(kappa=bad) == -1 and call(sigma=bad) == -1
    for k in range(K):                                                  # a bad entry of any pose
        for i in (0, 3, 11):
            p = (C.c_double * (16 * K))(*poses)
            p[16 * k + i] = float("nan")
            assert call(p=p) == -1
    p = (C.c_double * (16 * K))(*poses)
    p[16 * (K - 1) + 15] = float("inf")                                 # row 3 is not read ...
    assert call(p=p, o=_abi.ShineOctree()) == -1                        # ... but an empty octree is refused
    dec.hidden = 64
    assert call() == -2
    dec.hidden, oct_.feature_dim = 32, 6
    assert call() == -2
    # the scratch size: min(ceil(n / 256), 1024) blocks of 29 doubles per pose
    assert lib.shine_register_scratch_bytes(0, 5) == 0
    assert lib.shine_register_scratch_bytes(257, 2) == 2 * 2 * 29 * 8
    assert lib.shine_register_scratch_bytes(10 ** 6, 1105) == 1024 * 1105 * 29 * 8
    assert lib.shine_register_scratch_bytes(-1, 1) == -1 and lib.shine_register_scratch_bytes(1, 0) == -1


def test_launch_poses_batches_stay_within_the_scratch_bound(monkeypatch):
    """A 10^6-point scan and the full coarse grid: launch_poses hands the entry batches whose scratch fits
    SCRATCH_BOUND_BYTES, every pose once and in order, each into its own rows of out."""
    from shine_mapping_b200 import _abi
    from tests.parity_utils import make_config
    grid = (len(odometry.ScanToMapRegistration.GRID_X) * len(odometry.ScanToMapRegistration.GRID_Y) *
            len(odometry.ScanToMapRegistration.GRID_YAW))
    assert grid == 1105
    calls = []
    real = _abi.lib()

    class Lib:
        shine_register_scratch_bytes = staticmethod(real.shine_register_scratch_bytes)

        @staticmethod
        def shine_register_normal_eq_poses(od, dd, points, n, poses, kc, sigma, kappa, out, scratch, scratch_bytes, st):
            calls.append((n, kc, [poses[16 * k + 3] for k in range(kc)], out.value, scratch_bytes))
            return 0

    class Fake:
        """a CUDA tensor's surface as launch_poses uses it"""
        is_cuda = True
        device = torch.device("cuda:0")

        def __init__(self, n):
            self.shape = (n, 3)

        def float(self):
            return self

        def contiguous(self):
            return self

        def data_ptr(self):
            return 0

    class Registration(odometry.ScanToMapRegistration):
        def __init__(self):
            self.sigma, self.device = 1.0, torch.device("cuda:0")
            self.octree = type("O", (), {"_descriptor": lambda self, a, b: _abi.ShineOctree()})()
            self.decoder = type("D", (), {"c_descriptor": lambda self, a: _abi.ShineDecoder()})()
            self.scratch = _Buf(0)

    monkeypatch.setattr(_abi, "lib", lambda: Lib)
    monkeypatch.setattr(_abi, "stream_ptr", lambda dev: None)
    monkeypatch.setattr(torch, "empty", lambda n, dtype=None, device=None: _Buf(n))
    reg = Registration()
    poses = np.tile(np.eye(4), (grid, 1, 1))
    poses[:, 0, 3] = np.arange(grid)
    out = _Out(grid)
    reg.launch_poses(Fake(10 ** 6), poses, 0.1, out)
    per_pose = 1024 * 29 * 8
    assert [c[1] for c in calls] == [282, 282, 282, 259]
    assert all(c[0] == 10 ** 6 and c[4] >= c[1] * per_pose and c[1] * per_pose <= 64 << 20 for c in calls)
    assert [x for c in calls for x in c[2]] == list(range(grid))
    assert [c[3] for c in calls] == [8 + k0 * 29 * 8 for k0 in (0, 282, 564, 846)]
    assert reg.scratch.nbytes == 282 * per_pose
    # out must be fp64 [K, 29] and contiguous
    with pytest.raises(ValueError, match="fp64"):
        reg.launch_poses(Fake(10), poses[:2], 0.1, _Out(3))


class _Buf:
    def __init__(self, n):
        self.nbytes = n

    def numel(self):
        return self.nbytes

    def data_ptr(self):
        return 0


class _Out:
    """an fp64 [K, 29] CUDA tensor's surface: out[a:b] points at row a"""
    dtype = torch.float64
    device = torch.device("cuda:0")

    def __init__(self, K, base=8):
        self.shape, self.base = (K, 29), base

    def is_contiguous(self):
        return True

    def __getitem__(self, sl):
        return _Out(sl.stop - sl.start, self.base + sl.start * 29 * 8)

    def data_ptr(self):
        return self.base
