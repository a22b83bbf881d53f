"""`SHINEConfig` — attribute bag with the reference's names (reference utils/config.py:6-375) so the
reference's YAML files (`config/**/*.yaml`) and caller code work unchanged with this package.

Implementation is table driven: `_DEFAULTS` holds the knobs the hot path and its drop-in callers read,
`_YAML_MAP` maps `section.key` of the reference YAML schema (reference utils/config.py:206-359) to the
attribute.  Keys for subsystems that are out of scope here (open3d visualiser, mesher, dataset I/O) are
still accepted and stored so a reference YAML never fails to load.
"""
from __future__ import annotations

import os

import torch
import yaml

_DEFAULTS = dict(
    # setting
    name="dummy", output_root="", pc_path="", pose_path="", calib_path="", label_path="",
    load_model=False, model_path="/", first_frame_ref=True, begin_frame=0, end_frame=0, every_frame=1,
    seed=42, num_workers=12, device="cuda", gpu_id="0", dtype=torch.float32, pc_count_gpu_limit=500,
    global_shift_default=0.0,
    # process
    min_range=2.75, pc_radius=20.0, min_z=-10.0, max_z=30.0, rand_downsample=True, vox_down_m=0.03,
    rand_down_r=1.0, filter_noise=False, sor_nn=25, sor_std=2.5, estimate_normal=False,
    normal_radius_m=0.2, normal_max_nn=20, map_vox_down_m=0.05,
    # semantics (off on the hot path)
    semantic_on=False, sem_class_count=20, sem_label_decimation=1, filter_moving_object=False,
    # octree
    tree_level_world=10, tree_level_feat=4, leaf_vox_size=0.5, feature_dim=8, feature_std=0.05,
    poly_int_on=True, octree_from_surface_samples=True,
    # sampler
    surface_sample_range_m=0.5, surface_sample_n=5, free_sample_begin_ratio=0.3,
    free_sample_end_dist_m=0.5, free_sample_n=2, clearance_dist_m=0.3, clearance_sample_n=0,
    # incremental mapping
    continual_learning_reg=True, lambda_forget=1e5, cal_importance_weight_down_rate=2,
    window_replay_on=True, window_radius=50.0, occu_update_on=False,
    # decoder
    geo_mlp_level=2, geo_mlp_hidden_dim=32, geo_mlp_bias_on=True,
    sem_mlp_level=2, sem_mlp_hidden_dim=32, sem_mlp_bias_on=True, freeze_after_frame=20,
    # loss
    ray_loss=False, main_loss_type="sdf_bce", loss_reduction="mean", sigma_sigmoid_m=0.1,
    sigma_scale_constant=0.0, logistic_gaussian_ratio=0.55, proj_correction_on=False, predict_sdf=False,
    neus_loss_on=False, loss_weight_on=False, behind_dropoff_on=False, dropoff_min_sigma=1.0,
    dropoff_max_sigma=5.0, normal_loss_on=False, weight_n=0.01, ekional_loss_on=False, weight_e=0.1,
    consistency_loss_on=False, weight_c=1.0, consistency_count=1000, consistency_range=0.1,
    history_weight=1.0, weight_s=1.0, time_conditioned=False,
    # optimizer
    iters=200, opt_adam=True, bs=4096, lr=1e-3, weight_decay=0.0, adam_eps=1e-15,
    lr_level_reduce_ratio=1.0, lr_iters_reduce_ratio=0.1, lr_decay_step=[10000, 50000, 100000], dropout=0,
    # eval / meshing (stored only)
    wandb_vis_on=False, o3d_vis_on=True, eval_on=False, eval_outlier_thre=0.5, eval_freq_iters=100,
    vis_freq_iters=100, save_freq_iters=100, mesh_freq_frame=1, mc_res_m=0.1, pad_voxel=1,
    mc_with_octree=True, mc_query_level=8, mc_vis_level=1, mc_mask_on=True, mc_local=False,
    min_cluster_vertices=50, infer_bs=4096, occ_binary_mc=False, grid_loss_vis_on=False,
    mesh_vis_on=True, save_map=False,
    # derived
    scale=1.0, world_size=1.0,
)

# "section.key" of the reference YAML -> (attribute, cast)
_YAML_MAP = {
    "setting.name": ("name", None), "setting.output_root": ("output_root", None),
    "setting.pc_path": ("pc_path", None), "setting.pose_path": ("pose_path", None),
    "setting.calib_path": ("calib_path", None), "setting.label_path": ("label_path", None),
    "setting.load_model": ("load_model", None), "setting.model_path": ("model_path", None),
    "setting.first_frame_ref": ("first_frame_ref", None), "setting.begin_frame": ("begin_frame", None),
    "setting.end_frame": ("end_frame", None), "setting.every_frame": ("every_frame", None),
    "setting.device": ("device", None), "setting.gpu_id": ("gpu_id", None),
    # not read from YAML by the reference (utils/config.py:35 keeps the default 500); accepted here so a config can set it
    "setting.pc_count_gpu_limit": ("pc_count_gpu_limit", int),
    "process.min_range_m": ("min_range", None), "process.pc_radius_m": ("pc_radius", None),
    "process.rand_downsample": ("rand_downsample", None), "process.vox_down_m": ("vox_down_m", None),
    "process.rand_down_r": ("rand_down_r", None), "process.min_z_m": ("min_z", None),
    "sampler.surface_sample_range_m": ("surface_sample_range_m", None),
    "sampler.surface_sample_n": ("surface_sample_n", None),
    "sampler.free_sample_begin_ratio": ("free_sample_begin_ratio", None),
    "sampler.free_sample_end_dist_m": ("free_sample_end_dist_m", None),
    "sampler.free_sample_n": ("free_sample_n", None),
    "octree.tree_level_world": ("tree_level_world", None), "octree.tree_level_feat": ("tree_level_feat", None),
    "octree.leaf_vox_size": ("leaf_vox_size", None), "octree.feature_dim": ("feature_dim", None),
    "octree.poly_int_on": ("poly_int_on", None),
    "octree.octree_from_surface_samples": ("octree_from_surface_samples", None),
    "decoder.mlp_level": ("geo_mlp_level", None), "decoder.mlp_hidden_dim": ("geo_mlp_hidden_dim", None),
    "decoder.freeze_after_frame": ("freeze_after_frame", None),
    "loss.ray_loss": ("ray_loss", None), "loss.main_loss_type": ("main_loss_type", None),
    "loss.sigma_sigmoid_m": ("sigma_sigmoid_m", None), "loss.loss_weight_on": ("loss_weight_on", None),
    "loss.behind_dropoff_on": ("behind_dropoff_on", None), "loss.ekional_loss_on": ("ekional_loss_on", None),
    "loss.weight_e": ("weight_e", float),
    "continual.continual_learning_reg": ("continual_learning_reg", None),
    "continual.lambda_forget": ("lambda_forget", float),
    "continual.window_replay_on": ("window_replay_on", None),
    "continual.window_radius_m": ("window_radius", None),
    "optimizer.iters": ("iters", None), "optimizer.batch_size": ("bs", None),
    "optimizer.learning_rate": ("lr", float), "optimizer.weight_decay": ("weight_decay", float),
    "eval.wandb_vis_on": ("wandb_vis_on", None), "eval.o3d_vis_on": ("o3d_vis_on", None),
    "eval.vis_freq_iters": ("vis_freq_iters", None), "eval.save_freq_iters": ("save_freq_iters", None),
    "eval.mesh_freq_frame": ("mesh_freq_frame", None), "eval.mc_with_octree": ("mc_with_octree", None),
    "eval.mc_res_m": ("mc_res_m", None), "eval.mc_vis_level": ("mc_vis_level", None),
    "eval.mc_local": ("mc_local", None), "eval.save_map": ("save_map", None),
}


class SHINEConfig:
    def __init__(self, **overrides):
        for key, value in _DEFAULTS.items():
            setattr(self, key, list(value) if isinstance(value, list) else value)
        for key, value in overrides.items():
            if key not in _DEFAULTS:
                raise AttributeError(f"unknown SHINEConfig field {key!r}")
            setattr(self, key, value)
        if overrides:
            self.calculate_world_scale()

    def load(self, config_file: str) -> None:
        """Read a reference-schema YAML (reference utils/config.py:206-369); unknown keys are ignored."""
        with open(os.path.abspath(config_file)) as fh:
            doc = yaml.safe_load(fh) or {}
        for section, body in doc.items():
            if not isinstance(body, dict):
                continue
            for key, value in body.items():
                target = _YAML_MAP.get(f"{section}.{key}")
                if target is None:
                    continue
                attr, cast = target
                setattr(self, attr, cast(value) if cast else value)
        self.calculate_world_scale()
        self.infer_bs = self.bs * 16  # reference utils/config.py:365
        self.mc_query_level = self.tree_level_world - self.tree_level_feat + 1  # :366
        if self.window_radius <= 0:
            self.window_radius = self.pc_radius * 2.0

    def calculate_world_scale(self) -> None:
        """scale = 1 / (leaf_vox_size * 2^(tree_level_world-1)) maps metres into kaolin's [-1,1] cube
        (reference utils/config.py:372-374)."""
        self.world_size = self.leaf_vox_size * (2 ** (self.tree_level_world - 1))
        self.scale = 1.0 / self.world_size

    @property
    def sigma_sigmoid(self) -> float:
        """The fixed sigmoid width used by the BCE loss (reference shine_batch.py:87)."""
        return self.logistic_gaussian_ratio * self.sigma_sigmoid_m * self.scale
