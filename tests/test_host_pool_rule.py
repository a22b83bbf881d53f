"""The host sample pool without a GPU: the reference's rule for where the batch-mode pool lives, the YAML key that sets
its limit, the descriptor layout and the argument checks of the two entry points that run before any CUDA call."""
import ctypes as C

import pytest

from tests.parity_utils import make_config


def test_use_host_pool_states_the_reference_rule():
    from shine_mapping_b200 import synth
    cfg = make_config(2, continual_learning_reg=False, window_replay_on=False)
    assert cfg.pc_count_gpu_limit == 500                         # reference utils/config.py:35
    assert not synth.use_host_pool(cfg, 500)                     # strictly more scans than the limit
    assert synth.use_host_pool(cfg, 501)
    cfg.pc_count_gpu_limit = 2
    assert not synth.use_host_pool(cfg, 0) and not synth.use_host_pool(cfg, 2) and synth.use_host_pool(cfg, 3)
    # incremental modes keep the pool on the device whatever the count (dataset/lidar_dataset.py:94)
    assert not synth.use_host_pool(make_config(2, pc_count_gpu_limit=2, continual_learning_reg=True,
                                               window_replay_on=False), 3)
    assert not synth.use_host_pool(make_config(2, pc_count_gpu_limit=2, continual_learning_reg=False,
                                               window_replay_on=True), 3)
    assert not synth.use_host_pool(make_config(2, pc_count_gpu_limit=2), 3)     # both on by default


def test_yaml_sets_pc_count_gpu_limit(tmp_path):
    from shine_mapping_b200.config import SHINEConfig
    y = tmp_path / "c.yaml"
    y.write_text("setting: {name: x, pc_count_gpu_limit: 2}\n")
    cfg = SHINEConfig()
    cfg.load(str(y))
    assert cfg.pc_count_gpu_limit == 2
    y.write_text("setting: {name: x}\n")
    cfg = SHINEConfig()
    cfg.load(str(y))
    assert cfg.pc_count_gpu_limit == 500


def test_host_pool_struct_layout():
    from shine_mapping_b200 import _abi
    assert C.sizeof(_abi.ShineHostPool) == 24
    assert _abi.ShineHostPool.chunk_shift.offset == 8 and _abi.ShineHostPool.size.offset == 16


def test_host_pool_argument_checks_need_no_gpu(built_lib):
    from shine_mapping_b200 import _abi
    lib = built_lib
    table = (C.c_int64 * 4)()                   # placeholder: every call below returns before it is dereferenced
    good = _abi.ShineHostPool(C.addressof(table), 10, 4, 100)
    assert lib.shine_host_pool_append(None, 0, None, None, None, 0, None) == -1
    assert lib.shine_host_pool_gather(None, None, 0, None, None, None, None) == -1
    assert lib.shine_host_pool_append(C.byref(good), 0, None, None, None, 0, None) == 0        # nothing to do
    assert lib.shine_host_pool_gather(C.byref(good), None, 0, None, None, None, None) == 0
    assert lib.shine_host_pool_gather(C.byref(good), None, -1, None, None, None, None) == -1
    assert lib.shine_host_pool_append(C.byref(good), 0, None, None, None, -1, None) == -1
    assert lib.shine_host_pool_append(C.byref(good), -1, None, None, None, 0, None) == -1
    assert lib.shine_host_pool_append(C.byref(good), 4 << 10, None, None, None, 1, None) == -1  # past the last chunk
    assert lib.shine_host_pool_append(C.byref(good), 0, None, None, None, 1, None) == -1        # null frame buffers
    assert lib.shine_host_pool_gather(C.byref(good), None, 5, None, None, None, None) == -1     # null index / outputs
    for kw in (dict(chunks=None), dict(chunk_shift=4), dict(chunk_shift=32), dict(num_chunks=-1), dict(size=-1),
               dict(size=(4 << 10) + 1)):
        bad = _abi.ShineHostPool(C.addressof(table), 10, 4, 100)
        for k, v in kw.items():
            setattr(bad, k, v)
        assert lib.shine_host_pool_append(C.byref(bad), 0, None, None, None, 0, None) == -1, kw
        assert lib.shine_host_pool_gather(C.byref(bad), None, 0, None, None, None, None) == -1, kw
    assert lib.shine_error_string(-1).decode() == "shine_b200: invalid argument"


def test_build_scene_map_rejects_an_unknown_pool_mode():
    from shine_mapping_b200 import synth
    with pytest.raises(ValueError):
        synth.build_scene_map(make_config(2), None, 16, 1, pool="cpu")
