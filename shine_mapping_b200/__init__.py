"""shine_mapping_b200 — H100-native (sm_90a) implementation of SHINE-mapping's per-point SDF training step
behind the reference's own `FeatureOctree` / `Decoder` / `sdf_bce_loss` surfaces (see DESIGN.md)."""
from .config import SHINEConfig
from .decoder import Decoder
from .feature_octree import FeatureOctree
from .fused import sdf_bce_step, sdf_diff_step, sdf_infer
from .loss import sdf_bce_loss, sdf_diff_loss
from .mesher import Mesher
from .trainer import SdfTrainer

__all__ = ["SHINEConfig", "Decoder", "FeatureOctree", "sdf_bce_step", "sdf_diff_step", "sdf_infer", "sdf_bce_loss",
           "sdf_diff_loss", "SdfTrainer", "Mesher"]
