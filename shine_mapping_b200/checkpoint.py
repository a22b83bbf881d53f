"""Reading saved maps — the one module that knows the checkpoint formats (DESIGN.md §10).

Three kinds of `.pth` file are accepted, all `torch.save`d dicts with a `geo_decoder` state dict:

* this package's own (`batch_loop.save_checkpoint`): `feature_octree` is a pickled
  `shine_mapping_b200.feature_octree.FeatureOctree`;
* decoder-only files (the reference's `pretrained/geo_decoder_8dim.pth`, its `*_decoders.pth`): no `feature_octree`;
* the reference's (utils/tools.py:200-213): `feature_octree` is a pickled `model.feature_octree.FeatureOctree`, a class
  that does not exist here.  The unpickler maps that one name to a stand-in that only receives the module's state, and the
  map is rebuilt from its lookup dicts by `FeatureOctree.from_lookup_tables`.

`torch.load(..., weights_only=False)` executes pickles: checkpoints are TRUSTED input, as in the reference
(shine_batch.py:46).  The unpickler used here resolves the globals a map file needs (`_ALLOWED`) and refuses every other one
instead of importing it, which is what lets a reference file load without the reference; it is not a sandbox.
"""
from __future__ import annotations

import copy
import pickle
import types

import torch

from .config import SHINEConfig
from .decoder import Decoder
from .feature_octree import FeatureOctree


class _ReferenceOctree:
    """What a pickled `model.feature_octree.FeatureOctree` unpickles to: the nn.Module's `__dict__`, nothing else."""

    def __setstate__(self, state):
        self.__dict__.update(state)


_STORAGES = ("FloatStorage", "DoubleStorage", "HalfStorage", "BFloat16Storage", "LongStorage", "IntStorage", "ShortStorage",
             "CharStorage", "ByteStorage", "BoolStorage")
_ALLOWED = {("collections", "OrderedDict"), ("builtins", "set"),
            ("torch._utils", "_rebuild_tensor_v2"), ("torch._utils", "_rebuild_parameter"),
            ("torch._utils", "_rebuild_parameter_with_state"), ("torch", "device"), ("torch", "Size"),
            ("torch.nn.modules.container", "ParameterList"),
            ("shine_mapping_b200.feature_octree", "FeatureOctree"), ("shine_mapping_b200.feature_octree", "_LevelState"),
            *(("torch", s) for s in _STORAGES)}


class _Unpickler(pickle.Unpickler):
    def find_class(self, module, name):
        if (module, name) == ("model.feature_octree", "FeatureOctree"):
            return _ReferenceOctree
        if module == "__builtin__":          # protocol 2 files name the builtins the Python 2 way
            module = "builtins"
        if (module, name) in _ALLOWED:
            return super().find_class(module, name)
        raise pickle.UnpicklingError(f"the checkpoint names the global {module}.{name}, which no map file needs: refused")


# what torch.load takes as `pickle_module`
_PICKLE = types.SimpleNamespace(__name__="shine_mapping_b200.checkpoint", Unpickler=_Unpickler,
                                load=lambda f, **kw: _Unpickler(f, **kw).load())

# config attribute -> attribute of the octree: they fix `scale` and the kernels' template dispatch
_OCTREE_KEYS = (("tree_level_world", "max_level"), ("tree_level_feat", "featured_level_num"), ("feature_dim", "feature_dim"),
                ("poly_int_on", "polynomial_interpolation"), ("leaf_vox_size", "leaf_vox_size"))


def _check_octree_config(config: SHINEConfig, saved) -> None:
    for key, attr in _OCTREE_KEYS:
        if not hasattr(saved, attr):
            raise ValueError(f"{key}: the checkpoint's feature_octree has no {attr}")
        have, want = getattr(saved, attr), getattr(config, key)
        if have != want:
            raise ValueError(f"{key}: the checkpoint's map was built with {have!r}, the config says {want!r}")


def _check_decoder(config: SHINEConfig, state) -> None:
    if not isinstance(state, dict):
        raise ValueError("geo_decoder: not a state dict")
    cfg = copy.copy(config)
    cfg.device = "cpu"
    want = Decoder(cfg).state_dict()
    for key, t in want.items():
        if key not in state:
            raise ValueError(f"geo_decoder.{key}: missing from the checkpoint (the config's geo_mlp_level / geo_mlp_bias_on "
                             "ask for it)")
        if tuple(state[key].shape) != tuple(t.shape):
            raise ValueError(f"geo_decoder.{key}: the checkpoint holds {tuple(state[key].shape)}, the config (feature_dim, "
                             f"geo_mlp_hidden_dim, geo_mlp_level, sem_class_count) asks for {tuple(t.shape)}")
    extra = sorted(set(state) - set(want))
    if extra:
        raise ValueError(f"geo_decoder.{extra[0]}: not a parameter of the config's decoder (geo_mlp_level / geo_mlp_bias_on)")


def load_checkpoint(path: str, config: SHINEConfig, device):
    """-> (geo_decoder state dict, FeatureOctree on `device` or None when the file holds no map).

    `path` is unpickled (`weights_only=False`): load only files you trust.  The decoder's shapes and the map's
    `tree_level_world`, `tree_level_feat`, `feature_dim`, `poly_int_on`, `leaf_vox_size` must agree with `config`, and the
    map's tables must be consistent; each violation is a ValueError naming the key.  `sem_decoder`, `optimizer` and `iters`
    are left unread."""
    loaded = torch.load(path, map_location=device, pickle_module=_PICKLE, weights_only=False)
    if not isinstance(loaded, dict) or "geo_decoder" not in loaded:
        raise ValueError(f"{path}: not a checkpoint (no geo_decoder)")
    _check_decoder(config, loaded["geo_decoder"])
    saved = loaded.get("feature_octree")
    if saved is None:
        return loaded["geo_decoder"], None
    if not isinstance(saved, (FeatureOctree, _ReferenceOctree)):
        raise ValueError(f"{path}: feature_octree is a {type(saved).__name__}, not a map")
    _check_octree_config(config, saved)
    if isinstance(saved, FeatureOctree):
        octree = saved.to(device)
        if octree.is_empty():       # _apply takes the device from the tables
            octree.device = device
        octree.check_tables()
        return loaded["geo_decoder"], octree
    cfg = copy.copy(config)
    cfg.device = device
    state = saved.__dict__
    try:
        tables = [p.data for p in state["_modules"]["hier_features"]]
        corners, nodes = state["corners_lookup_tables"], state["nodes_lookup_tables"]
    except (KeyError, TypeError) as e:
        raise ValueError(f"{path}: feature_octree lacks {e}") from None
    octree = FeatureOctree.from_lookup_tables(cfg, corners, nodes, tables, state.get("importance_weight", ()),
                                              state.get("features_last_frame", ()))
    return loaded["geo_decoder"], octree


def apply_load_model(config: SHINEConfig, octree: FeatureOctree, decoder: Decoder) -> FeatureOctree:
    """`setting.load_model` (shine_batch.py:45-55, shine_incre.py:44-54): load `config.model_path`, put its geo decoder into
    `decoder` and freeze it (utils/tools.py:188-191), and return the file's map when it holds one, else `octree`.  With
    `load_model` off, `octree` comes back untouched."""
    if not config.load_model:
        return octree
    state, loaded = load_checkpoint(config.model_path, config, next(decoder.parameters()).device)
    decoder.load_state_dict(state)
    for child in decoder.children():
        for p in child.parameters():
            p.requires_grad = False
    print("Pretrained decoder loaded")
    if loaded is None:
        return octree
    loaded.print_detail()
    return loaded
