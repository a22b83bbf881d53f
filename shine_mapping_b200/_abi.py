"""ctypes binding of the C ABI in include/shine_b200.h (csrc/libshine_b200.so).

There is no fallback: if the library is missing or a call fails, an exception is raised.  The library is
built in-tree by `__graft_entry__.build()` (nvcc, sm_90a).
"""
from __future__ import annotations

import ctypes as C
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("SHINE_B200_LIB") or os.path.join(_HERE, "csrc", "libshine_b200.so")

ABI_VERSION = 5
MAX_LEVELS = 8
HASH_SLOT_BYTES = 64
ADAM_MAX_TENSORS = 16
FLAG_REDUCTION_SUM = 1
FLAG_WEIGHTED = 2
FLAG_TF32X1 = 4
FLAG_MORTON_ORDERED = 16
FLAG_LOSS_L2 = 32
FLAG_LOSS_L1 = 64
ERR_CAPACITY = -3
REGISTER_OUT = 29
REGISTER_SCRATCH_BYTES = 1024 * REGISTER_OUT * 8
RAYCAST_MAX_REFINE = 32


class ShineLevel(C.Structure):
    _fields_ = [("hash_slots", C.c_void_p), ("features", C.c_void_p), ("feature_grads", C.c_void_p),
                ("grad_replicas", C.c_void_p),
                ("hash_capacity", C.c_uint32), ("rows", C.c_int32), ("level", C.c_int32), ("num_replicas", C.c_int32)]


class ShineOctree(C.Structure):
    _fields_ = [("num_levels", C.c_int32), ("feature_dim", C.c_int32), ("poly_interp", C.c_int32),
                ("reserved", C.c_int32), ("lv", ShineLevel * MAX_LEVELS)]


class ShineDecoder(C.Structure):
    _fields_ = [("w1", C.c_void_p), ("b1", C.c_void_p), ("w2", C.c_void_p), ("b2", C.c_void_p),
                ("w3", C.c_void_p), ("b3", C.c_void_p),
                ("gw1", C.c_void_p), ("gb1", C.c_void_p), ("gw2", C.c_void_p), ("gb2", C.c_void_p),
                ("gw3", C.c_void_p), ("gb3", C.c_void_p),
                ("in_dim", C.c_int32), ("hidden", C.c_int32), ("mlp_level", C.c_int32), ("reserved", C.c_int32)]


class ShineAdamTensor(C.Structure):
    _fields_ = [("param", C.c_void_p), ("grad", C.c_void_p), ("exp_avg", C.c_void_p), ("exp_avg_sq", C.c_void_p),
                ("numel", C.c_int64), ("lr", C.c_float), ("weight_decay", C.c_float)]


class ShineTouchedLevel(C.Structure):
    _fields_ = [("bitmap", C.c_void_p), ("rows", C.c_void_p), ("count", C.c_void_p), ("capacity", C.c_int32),
                ("reserved", C.c_int32)]


class ShineTouched(C.Structure):
    _fields_ = [("lv", ShineTouchedLevel * MAX_LEVELS)]


class ShineRowTables(C.Structure):
    _fields_ = [("last", C.c_void_p * MAX_LEVELS), ("importance", C.c_void_p * MAX_LEVELS),
                ("importance_rw", C.c_void_p * MAX_LEVELS)]


class ShineBoundaryLevel(C.Structure):
    _fields_ = [("table", C.c_void_p), ("rows", C.c_void_p), ("slots", C.c_void_p), ("offset", C.c_int64),
                ("count", C.c_int32), ("reserved", C.c_int32)]


class ShineBoundary(C.Structure):
    _fields_ = [("lv", ShineBoundaryLevel * MAX_LEVELS)]


class ShineBuildLevel(C.Structure):
    _fields_ = [("node_slots", C.c_void_p), ("corner_slots", C.c_void_p), ("frame_node_set", C.c_void_p),
                ("frame_corner_set", C.c_void_p), ("node_ids_out", C.c_void_p),
                ("corner_morton_out", C.c_void_p),
                ("node_capacity", C.c_uint32), ("corner_capacity", C.c_uint32), ("frame_node_set_capacity", C.c_uint32),
                ("frame_corner_set_capacity", C.c_uint32),
                ("level", C.c_int32), ("nodes_before", C.c_int32), ("rows_before", C.c_int32), ("reserved", C.c_int32)]


class ShineBuild(C.Structure):
    _fields_ = [("num_levels", C.c_int32), ("max_level", C.c_int32), ("new_node_count", C.c_void_p),
                ("new_corner_count", C.c_void_p), ("new_corner_total", C.c_void_p), ("new_node_total", C.c_void_p),
                ("new_node_keys", C.c_void_p), ("new_corner_keys", C.c_void_p),
                ("lv", ShineBuildLevel * MAX_LEVELS)]


class ShineBoundaryInverse(C.Structure):
    _fields_ = [("row_of_slot", C.c_void_p * MAX_LEVELS), ("slots", C.c_int32 * MAX_LEVELS),
                ("holders", C.c_void_p * MAX_LEVELS)]


class ShineSamplePool(C.Structure):
    _fields_ = [("coord", C.c_void_p), ("label", C.c_void_p), ("weight", C.c_void_p), ("size", C.c_int64),
                ("capacity", C.c_int64)]


class ShineHostPool(C.Structure):
    _fields_ = [("chunks", C.c_void_p), ("chunk_shift", C.c_int32), ("num_chunks", C.c_int32), ("size", C.c_int64)]


class ShineScanInput(C.Structure):
    _fields_ = [("records", C.c_void_p), ("n", C.c_int64), ("stride_bytes", C.c_int32), ("fp64", C.c_int32)]


class ShineBrickGrid(C.Structure):
    _fields_ = [("bricks", C.c_void_p), ("sdf", C.c_void_p), ("mask", C.c_void_p), ("all_keys", C.c_void_p),
                ("num_all", C.c_int64), ("num_bricks", C.c_int64), ("origin", C.c_float * 3), ("spacing", C.c_float),
                ("n", C.c_int32), ("lo", C.c_int32 * 3), ("hi", C.c_int32 * 3), ("missing_sdf", C.c_float)]


# name -> (restype, argtypes); every symbol declared in include/shine_b200.h
_vp, _i64, _i32, _u32, _f32 = C.c_void_p, C.c_int64, C.c_int32, C.c_uint32, C.c_float
_OCT, _DEC = C.POINTER(ShineOctree), C.POINTER(ShineDecoder)
SYMBOLS = {
    "shine_abi_version": (C.c_int, []),
    "shine_error_string": (C.c_char_p, [C.c_int]),
    "shine_hash_insert": (C.c_int, [_vp, _u32, _vp, _vp, _i64, _i32, _vp, _vp]),
    "shine_points_to_morton": (C.c_int, [_vp, _i64, _i32, _vp, _vp]),
    "shine_get_indices": (C.c_int, [_OCT, _vp, _i64, _vp, _vp]),
    "shine_query_fwd": (C.c_int, [_OCT, _vp, _i64, _vp, _vp]),
    "shine_query_bwd": (C.c_int, [_OCT, _vp, _i64, _vp, _vp]),
    "shine_query_coord_grad": (C.c_int, [_OCT, _vp, _i64, _vp, _vp, _vp]),
    "shine_query_tangent_fwd": (C.c_int, [_OCT, _vp, _i64, _vp, _vp, _vp]),
    "shine_query_tangent_bwd": (C.c_int, [_OCT, _vp, _i64, _vp, _vp, _vp]),
    "shine_sdf_infer": (C.c_int, [_OCT, _DEC, _vp, _i64, _vp, _vp, _i32, _u32, _vp]),
    "shine_sdf_fwd": (C.c_int, [_OCT, _DEC, _vp, _vp, _vp, _i64, _f32, _f32, _f32, _vp, _vp, _u32, _vp]),
    "shine_sdf_step": (C.c_int, [_OCT, _DEC, _vp, _vp, _vp, _i64, _f32, _f32, _f32, _vp, _vp, _vp, _u32, _vp]),
    "shine_sdf_bce_fwd": (C.c_int, [_OCT, _DEC, _vp, _vp, _vp, _i64, _f32, _f32, _vp, _vp, _u32, _vp]),
    "shine_reduce_grad_replicas": (C.c_int, [_OCT, _vp]),
    "shine_octree_frame_nodes": (C.c_int, [C.POINTER(ShineBuild), _vp, _i64, _vp]),
    "shine_octree_frame_corners": (C.c_int, [C.POINTER(ShineBuild), _i32, _vp]),
    "shine_octree_sort_scratch_bytes": (C.c_int64, [_i32]),
    "shine_octree_sort_new_keys": (C.c_int, [_vp, _vp, _i32, _vp, _i64, _vp]),
    "shine_octree_assign_rows": (C.c_int, [C.POINTER(ShineBuild), _vp, _i32, _vp]),
    "shine_octree_fill_nodes": (C.c_int, [C.POINTER(ShineBuild), _vp, _i32, _vp, _vp]),
    "shine_octree_corner_rehash": (C.c_int, [_vp, _u32, _vp, _i64, _vp]),
    "shine_count_positive": (C.c_int, [_vp, _i64, _vp, _vp]),
    "shine_sdf_eikonal_step": (C.c_int, [_OCT, _DEC, _vp, _vp, _vp, _i64, _f32, _f32, _f32, _f32, _vp, _vp, _vp, _vp, _vp,
                                         _u32, _vp]),
    "shine_mark_touched": (C.c_int, [_OCT, _vp, _i64, C.POINTER(ShineTouched), _vp]),
    "shine_regularization_apply": (C.c_int, [_OCT, C.POINTER(ShineTouched), C.POINTER(ShineRowTables), _f32, _vp, _i32, _vp]),
    "shine_importance_accumulate": (C.c_int, [_OCT, C.POINTER(ShineTouched), C.POINTER(ShineRowTables), _i32, _i32, _vp]),
    "shine_boundary_pack": (C.c_int, [C.POINTER(ShineBoundary), _i32, _i32, _vp, _vp]),
    "shine_boundary_unpack": (C.c_int, [C.POINTER(ShineBoundary), _i32, _i32, _vp, _vp]),
    "shine_nccl_unique_id": (C.c_int, [_vp]),
    "shine_nccl_comm_create": (C.c_int, [_vp, _i32, _i32, _i32, C.POINTER(C.c_void_p)]),
    "shine_nccl_comm_destroy": (C.c_int, [_vp]),
    "shine_allreduce_decoder_grads": (C.c_int, [_vp, _vp, _i64, _vp]),
    "shine_comm_last_error": (C.c_char_p, []),
    "shine_p2p_create": (C.c_int, [_i32, _i32, _i32, _i64, _vp, C.POINTER(C.c_void_p)]),
    "shine_p2p_connect": (C.c_int, [_vp, _vp]),
    "shine_p2p_exchange": (C.c_int, [_vp, _vp, _i64, C.POINTER(ShineBoundary), C.POINTER(ShineBoundaryInverse), _i32, _i32, _vp]),
    "shine_p2p_timeouts": (C.c_int, [_vp, C.POINTER(C.c_int32)]),
    "shine_p2p_destroy": (C.c_int, [_vp]),
    "shine_adam_step": (C.c_int, [C.POINTER(ShineAdamTensor), _i32, _f32, _f32, _f32, _i32, _i32, _vp]),
    "shine_adam_step_dev": (C.c_int, [C.POINTER(ShineAdamTensor), _i32, _f32, _f32, _f32, _vp, _i32, _vp]),
    "shine_pool_scratch_bytes": (C.c_int64, [_i64]),
    "shine_pool_window_append": (C.c_int, [C.POINTER(ShineSamplePool), _vp, _vp, _vp, _i64, _f32, _f32, _f32, _f32, _vp,
                                           _vp, _i64, _vp]),
    "shine_host_pool_append": (C.c_int, [C.POINTER(ShineHostPool), _i64, _vp, _vp, _vp, _i64, _vp]),
    "shine_host_pool_gather": (C.c_int, [C.POINTER(ShineHostPool), _vp, _i64, _vp, _vp, _vp, _vp]),
    "shine_scan_scratch_bytes": (C.c_int64, [_i64]),
    "shine_scan_filter_keys": (C.c_int, [C.POINTER(ShineScanInput), C.c_double, C.c_double, C.c_double, C.c_double,
                                         C.c_double, _vp, _i64, _vp]),
    "shine_scan_sort_voxels": (C.c_int, [_i64, _vp, _vp, _i64, _vp]),
    "shine_scan_average_transform": (C.c_int, [C.POINTER(ShineScanInput), C.POINTER(C.c_double), C.c_double, _i64, _vp,
                                               _vp, _vp, _i64, _vp]),
    "shine_scan_sample": (C.c_int, [_vp, _i64, _f32, _f32, _f32, _vp, _i32, _vp, _i32, _f32, _f32, _f32, _vp, _vp, _vp,
                                    _vp]),
    "shine_rgbd_backproject": (C.c_int, [_vp, _i32, _i32, _i32, C.c_double, C.c_double, C.c_double, C.c_double,
                                         C.c_double, C.c_double, C.POINTER(C.c_double), _vp, _vp, _vp, _vp]),
    "shine_mesh_grid": (C.c_int, [_OCT, _DEC, C.POINTER(ShineBrickGrid), _i32, _u32, _vp]),
    "shine_marching_cubes": (C.c_int, [C.POINTER(ShineBrickGrid), _vp, _u32, _vp, _vp, _i64, _vp, _i64, _vp]),
    "shine_mesh_export_points": (C.c_int, [C.POINTER(ShineBrickGrid), C.POINTER(C.c_double), C.c_double,
                                           C.POINTER(C.c_double), _f32, _i32, _vp, _i64, _vp, C.POINTER(_i64), _vp]),
    "shine_mesh_clusters": (C.c_int, [_vp, _i64, _vp, _i64, _i32, _vp, _u32, _vp, _vp, _vp, _vp]),
    "shine_mesh_sample_scratch_bytes": (C.c_int64, [_i64]),
    "shine_mesh_sample_areas": (C.c_int, [_vp, _i64, _vp, _i64, _vp, _vp, _vp, _i64, _vp]),
    "shine_mesh_sample_points": (C.c_int, [_vp, _vp, _i64, _vp, _i64, C.c_uint64, _vp, _i64, _vp, _vp, _vp]),
    "shine_nn_tree_bytes": (C.c_int64, [_i64]),
    "shine_nn_scratch_bytes": (C.c_int64, [_i64]),
    "shine_nn_build": (C.c_int, [_vp, _i64, _vp, _i64, _vp, _i64, _vp]),
    "shine_nn_query": (C.c_int, [_vp, _i64, _vp, _i64, C.c_double, _vp, _vp, _vp, _i64, _vp]),
    "shine_register_normal_eq": (C.c_int, [_OCT, _DEC, _vp, _i64, C.POINTER(C.c_double), _f32, C.c_double, _vp, _vp,
                                           _i64, _vp]),
    "shine_register_scratch_bytes": (C.c_int64, [_i64, _i64]),
    "shine_register_normal_eq_poses": (C.c_int, [_OCT, _DEC, _vp, _i64, C.POINTER(C.c_double), _i64, _f32, C.c_double,
                                                 _vp, _vp, _i64, _vp]),
    "shine_raycast": (C.c_int, [_OCT, _DEC, C.POINTER(_f32), _vp, _i64, _f32, _f32, _f32, _f32, _i32, _i32, _vp, _vp,
                                _vp]),
}

_lib = None


class ShineB200Error(RuntimeError):
    pass


def lib() -> C.CDLL:
    """Load csrc/libshine_b200.so (once).  Raises if it has not been built — no CPU / eager fallback."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ShineB200Error(
                f"{LIB_PATH} is missing: build the sm_90a kernels first (python -c 'import __graft_entry__ as g; "
                "g.build()').  shine_mapping_b200 has no CPU or eager fallback for the hot path.")
        handle = C.CDLL(LIB_PATH)
        for name, (restype, argtypes) in SYMBOLS.items():
            fn = getattr(handle, name)
            fn.restype, fn.argtypes = restype, argtypes
        if handle.shine_abi_version() != ABI_VERSION:
            raise ShineB200Error("libshine_b200.so ABI version mismatch; rebuild")
        _lib = handle
    return _lib


LAUNCHES = {"count": 0}   # successful kernel-launching ABI calls (bench.py reports it as gpu_launches)


def check(rc: int, what: str) -> None:
    LAUNCHES["count"] += 1
    if rc != 0:
        msg = (lib().shine_comm_last_error() if rc <= -1000 else lib().shine_error_string(rc)).decode()
        raise ShineB200Error(f"{what} failed: {msg} (code {rc})")


def require_cuda(t: torch.Tensor, what: str) -> None:
    if not t.is_cuda:
        raise ShineB200Error(
            f"{what}: tensor is on {t.device}; the hot path runs only as sm_90a CUDA kernels (no CPU fallback)")


def ptr(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def stream_ptr(device=None):
    return C.c_void_p(torch.cuda.current_stream(device).cuda_stream)
