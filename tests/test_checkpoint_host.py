"""Loading saved maps on the host (shine_mapping_b200/checkpoint.py, FeatureOctree.from_lookup_tables): the reference-written
fixture tests/golden/ref_checkpoint_l3.pt (minted by oracle/make_checkpoint_golden.py) without the reference, the inverse of
the dict views, decoder-only files, and every check on what a file may hold."""
import copy
import importlib.util
import io
import json
import os
import pickle
import sys

import numpy as np
import pytest
import torch

from shine_mapping_b200 import checkpoint
from shine_mapping_b200.config import SHINEConfig
from shine_mapping_b200.decoder import Decoder
from shine_mapping_b200.feature_octree import FeatureOctree

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
LEVEL_ARRAYS = ("node_keys", "node_ids", "node_keys_sorted", "corner_lex_sorted", "corner_rows_sorted", "corner_morton_by_row")


def _fixture():
    g = np.load(os.path.join(GOLD, "ref_checkpoint_l3.npz"))
    cfg = SHINEConfig(device="cpu", **json.loads(str(g["cfg_json"])))
    return g, cfg, os.path.join(GOLD, "ref_checkpoint_l3.pt")


def _grown(levels, frames=3, seed=0):
    torch.manual_seed(seed)
    cfg = SHINEConfig(device="cpu", tree_level_world=10, tree_level_feat=levels, leaf_vox_size=0.2)
    octree = FeatureOctree(cfg)
    clouds = [(torch.rand(400, 3) - 0.5) * 0.05 + 0.01 * f for f in range(frames + 1)]
    for c in clouds[:frames]:
        octree.update(c, incremental_on=True)
    return cfg, octree, clouds[frames]


def _save(tmp_path, cfg, octree=None, decoder=None, name="ckpt.pth", **extra):
    decoder = decoder or Decoder(cfg)
    d = {"geo_decoder": decoder.state_dict(), **extra}
    if octree is not None:
        d["feature_octree"] = octree
    path = str(tmp_path / name)
    torch.save(d, path)
    return path, decoder


def test_reference_checkpoint_loads_without_the_reference():
    g, cfg, path = _fixture()
    assert not any("reference" in p for p in sys.path)
    assert importlib.util.find_spec("model") is None and "model" not in sys.modules
    state, octree = checkpoint.load_checkpoint(path, cfg, "cpu")
    assert "model" not in sys.modules and isinstance(octree, FeatureOctree)
    assert set(state) == set(Decoder(cfg).state_dict())
    seen = 0
    for lvl in range(cfg.tree_level_world + 1):
        nodes, corners = octree.nodes_lookup_tables[lvl], octree.corners_lookup_tables[lvl]
        if f"node_keys_{lvl}" not in g:
            assert not nodes and not corners
            continue
        seen += 1
        assert list(nodes.keys()) == g[f"node_keys_{lvl}"].tolist()          # content and order
        assert list(nodes.values()) == g[f"node_ids_{lvl}"].tolist()
        assert list(corners.keys()) == g[f"corner_keys_{lvl}"].tolist()
        assert list(corners.values()) == g[f"corner_rows_{lvl}"].tolist()
    assert seen == cfg.tree_level_feat
    for k, p in enumerate(octree.hier_features):
        assert p.dtype == torch.float32 and p.detach().numpy().tobytes() == g[f"table_{k}"].tobytes()
    # the fixture's map was grown with incremental_on: the regularisation tables come along
    assert [tuple(t.shape) for t in octree.importance_weight] == [tuple(p.shape) for p in octree.hier_features]
    assert [tuple(t.shape) for t in octree.features_last_frame] == [tuple(p.shape) for p in octree.hier_features]


class _Evil:
    def __reduce__(self):
        return (os.getcwd, ())


@pytest.mark.parametrize("payload", [_Evil(), pickle.Unpickler, np.float32(1.0)])
def test_any_other_global_is_refused(tmp_path, payload):
    cfg = SHINEConfig(device="cpu")
    path = str(tmp_path / "crafted.pth")
    torch.save({"geo_decoder": Decoder(cfg).state_dict(), "feature_octree": None, "extra": payload}, path)
    with pytest.raises(pickle.UnpicklingError, match="refused"):
        checkpoint.load_checkpoint(path, cfg, "cpu")
    # and directly, whatever the container
    with pytest.raises(pickle.UnpicklingError, match="os|posix"):
        checkpoint._Unpickler(io.BytesIO(pickle.dumps(_Evil(), protocol=2))).load()


@pytest.mark.parametrize("levels", [1, 2, 3, 4])
def test_from_lookup_tables_inverts_the_dict_views(levels):
    cfg, octree, more = _grown(levels)
    rebuilt = FeatureOctree.from_lookup_tables(cfg, octree.corners_lookup_tables, octree.nodes_lookup_tables,
                                               [p.data for p in octree.hier_features], octree.importance_weight,
                                               octree.features_last_frame)
    def same(a, b):
        for sa, sb in zip(a._levels, b._levels):
            for name in LEVEL_ARRAYS:
                x, y = getattr(sa, name), getattr(sb, name)
                assert x.dtype == y.dtype and torch.equal(x, y), name
        assert len(a.hier_features) == len(b.hier_features) == levels
        for p, q in zip(a.hier_features, b.hier_features):
            assert torch.equal(p.data, q.data)
        for name in ("importance_weight", "features_last_frame"):
            assert all(torch.equal(x, y) for x, y in zip(getattr(a, name), getattr(b, name), strict=True))
        assert a.nodes_lookup_tables == b.nodes_lookup_tables and a.corners_lookup_tables == b.corners_lookup_tables
    same(octree, rebuilt)
    assert sum(st.node_keys.numel() for st in octree._levels) > 50
    before = [p.shape[0] for p in octree.hier_features]
    for o in (octree, rebuilt):          # one more frame on each: the same new nodes, rows and random features
        torch.manual_seed(99)
        o.update(more, incremental_on=True)
    assert [p.shape[0] for p in octree.hier_features] != before
    same(octree, rebuilt)


def test_own_checkpoint_round_trip_on_the_host(tmp_path):
    cfg, octree, _ = _grown(3)
    path, dec = _save(tmp_path, cfg, octree, iters=7, optimizer={"exp_avg": torch.zeros(4), "step": 3})
    state, loaded = checkpoint.load_checkpoint(path, cfg, "cpu")
    assert loaded is not octree and loaded.nodes_lookup_tables == octree.nodes_lookup_tables
    assert all(torch.equal(p.data, q.data) for p, q in zip(loaded.hier_features, octree.hier_features, strict=True))
    assert all(torch.equal(state[k], v) for k, v in dec.state_dict().items())


def test_decoder_only_file_freezes_the_decoder_and_keeps_the_octree(tmp_path, capsys):
    cfg, octree, _ = _grown(2)
    torch.manual_seed(5)
    path, saved = _save(tmp_path, cfg, sem_decoder={"anything": torch.zeros(1)})
    cfg.load_model, cfg.model_path = True, path
    dec = Decoder(cfg)
    assert not torch.equal(dec.lout.weight, saved.lout.weight)
    out = checkpoint.apply_load_model(cfg, octree, dec)
    assert out is octree
    assert all(torch.equal(v, saved.state_dict()[k]) for k, v in dec.state_dict().items())
    assert not any(p.requires_grad for p in dec.parameters())
    assert "Pretrained decoder loaded" in capsys.readouterr().out


def test_load_model_off_touches_nothing(tmp_path):
    cfg, octree, _ = _grown(2)
    cfg.load_model, cfg.model_path = False, str(tmp_path / "does_not_exist.pth")
    dec = Decoder(cfg)
    before = copy.deepcopy(dec.state_dict())
    assert checkpoint.apply_load_model(cfg, octree, dec) is octree
    assert all(torch.equal(v, before[k]) for k, v in dec.state_dict().items())
    assert all(p.requires_grad for p in dec.parameters())


def test_full_checkpoint_replaces_the_octree(tmp_path, capsys):
    cfg, octree, _ = _grown(2)
    path, _ = _save(tmp_path, cfg, octree)
    cfg.load_model, cfg.model_path = True, path
    fresh = FeatureOctree(cfg)
    out = checkpoint.apply_load_model(cfg, fresh, Decoder(cfg))
    assert out is not fresh and out.nodes_lookup_tables == octree.nodes_lookup_tables
    assert "Current Octomap" in capsys.readouterr().out


@pytest.mark.parametrize("field,value,key", [("geo_mlp_hidden_dim", 64, "geo_decoder.layers.0.weight"),
                                             ("feature_dim", 16, "geo_decoder.layers.0.weight"),
                                             ("geo_mlp_level", 3, "geo_decoder.layers.2.weight"),
                                             ("geo_mlp_level", 1, "geo_decoder.layers.1.bias"),
                                             ("geo_mlp_bias_on", False, "geo_decoder.layers.0.bias")])
def test_decoder_mismatch_names_the_key(tmp_path, field, value, key):
    cfg = SHINEConfig(device="cpu")
    path, _ = _save(tmp_path, cfg)
    other = SHINEConfig(device="cpu", **{field: value})
    with pytest.raises(ValueError, match=key.replace(".", r"\.")) as e:
        checkpoint.load_checkpoint(path, other, "cpu")
    if field == "geo_mlp_hidden_dim":
        assert "(32, 8)" in str(e.value) and "(64, 8)" in str(e.value)       # both shapes


_OCTREE_MISMATCH = [("tree_level_world", 11), ("tree_level_feat", 2), ("poly_int_on", False), ("leaf_vox_size", 0.25)]


# feature_dim on our own format only: the reference fixture's decoder disagrees first and names its own key
@pytest.mark.parametrize("field,value,ours", [(f, v, o) for o in (True, False) for f, v in _OCTREE_MISMATCH]
                         + [("feature_dim", 4, True)])
def test_octree_config_mismatch_names_the_key(tmp_path, field, value, ours):
    if ours:
        cfg, octree, _ = _grown(3)
    else:
        _, cfg, path = _fixture()
        _, octree = checkpoint.load_checkpoint(path, cfg, "cpu")
    other = copy.copy(cfg)
    setattr(other, field, value)
    other.calculate_world_scale()
    if ours:      # the decoder is the other config's, so that only the map disagrees with it
        path, _ = _save(tmp_path, other, octree)
    with pytest.raises(ValueError, match=f"{field}: the checkpoint's map"):
        checkpoint.load_checkpoint(path, other, "cpu")


def _tables(octree):
    return ([dict(d) for d in octree.corners_lookup_tables], [dict(d) for d in octree.nodes_lookup_tables],
            [p.data for p in octree.hier_features])


def test_tables_from_outside_are_checked():
    cfg, octree, _ = _grown(2)
    lvl = cfg.tree_level_world
    rows = octree.hier_features[-1].shape[0] - 1
    key = next(iter(octree.nodes_lookup_tables[lvl]))
    for bad in (rows, rows + 7, -1, -5, 2 ** 40):      # the trash row, past the table, a miss marker, negative, not an int32
        corners, nodes, tables = _tables(octree)
        nodes[lvl][key] = [bad] + nodes[lvl][key][1:]
        with pytest.raises(ValueError, match=f"nodes_lookup_tables level {lvl}"):
            FeatureOctree.from_lookup_tables(cfg, corners, nodes, tables)
    corners, nodes, tables = _tables(octree)
    nodes[lvl][key] = nodes[lvl][key][:7]
    with pytest.raises(ValueError, match="8 corner rows"):
        FeatureOctree.from_lookup_tables(cfg, corners, nodes, tables)
    corners, nodes, tables = _tables(octree)
    nodes[lvl][8 ** lvl] = nodes[lvl][key]
    with pytest.raises(ValueError, match="Morton code outside"):
        FeatureOctree.from_lookup_tables(cfg, corners, nodes, tables)
    corners, nodes, tables = _tables(octree)
    corners[lvl][next(iter(corners[lvl]))] = 1
    with pytest.raises(ValueError, match=f"corners_lookup_tables level {lvl}"):
        FeatureOctree.from_lookup_tables(cfg, corners, nodes, tables)
    corners, nodes, tables = _tables(octree)
    with pytest.raises(ValueError, match="corners_lookup_tables"):
        FeatureOctree.from_lookup_tables(cfg, corners, nodes, [tables[0], tables[1][:-3]])
    with pytest.raises(ValueError, match="hier_features"):
        FeatureOctree.from_lookup_tables(cfg, corners, nodes, tables[:1])
    with pytest.raises(ValueError, match="hier_features"):
        FeatureOctree.from_lookup_tables(cfg, corners, nodes, [tables[0], tables[1].double()])
    with pytest.raises(ValueError, match="importance_weight"):
        FeatureOctree.from_lookup_tables(cfg, corners, nodes, tables, importance_weight=[tables[0]])
    nodes[3] = {0: list(range(8))}
    with pytest.raises(ValueError, match="level 3"):
        FeatureOctree.from_lookup_tables(cfg, corners, nodes, tables)


def test_own_checkpoint_with_a_row_out_of_range_is_rejected(tmp_path):
    cfg, octree, _ = _grown(2)
    st = octree._levels[cfg.tree_level_world]
    st.node_ids[0, 0] = octree.hier_features[-1].shape[0] + 3
    path, _ = _save(tmp_path, cfg, octree)
    with pytest.raises(ValueError, match=f"nodes_lookup_tables level {cfg.tree_level_world}"):
        checkpoint.load_checkpoint(path, cfg, "cpu")


def test_not_a_checkpoint(tmp_path):
    cfg = SHINEConfig(device="cpu")
    path = str(tmp_path / "x.pth")
    torch.save({"iters": 3}, path)
    with pytest.raises(ValueError, match="geo_decoder"):
        checkpoint.load_checkpoint(path, cfg, "cpu")
    torch.save({"geo_decoder": Decoder(cfg).state_dict(), "feature_octree": {"a": 1}}, path)
    with pytest.raises(ValueError, match="feature_octree"):
        checkpoint.load_checkpoint(path, cfg, "cpu")


def test_sdf_map_header_is_fixed_width_and_reads_back(tmp_path):
    from shine_mapping_b200 import mesher
    assert len(mesher._SDF_MAP_HEADER.format(0)) == len(mesher._SDF_MAP_HEADER.format(10 ** 11))
    assert mesher.SDF_MAP_RECORD.itemsize == 20
    rec = np.zeros(5, dtype=mesher.SDF_MAP_RECORD)
    rec["x"], rec["intensities"], rec["labels"] = np.arange(5), -0.25, [0, 1, 1, 0, 1]
    path = str(tmp_path / "m.ply")
    with open(path, "wb") as fh:
        fh.write(mesher._SDF_MAP_HEADER.format(5).encode())
        fh.write(rec.tobytes())
    back = mesher.read_point_ply(path)
    assert back.dtype.names == ("x", "y", "z", "intensities", "labels") and np.array_equal(back, rec)
    from shine_mapping_b200.scans import read_ply
    assert read_ply(path, pinned=False).n == 5          # the scan reader takes the file as a point cloud too
