"""CPU-side tests: host logic of the package (octree growth, config, pickling, decoder surface), that the C-ABI
library loads and exports every symbol of include/shine_b200.h, and that the product path refuses to run on CPU."""
import os
import pickle
import re

import numpy as np
import pytest
import torch

from tests.parity_utils import GOLDEN_NAMES, ROOT, load_golden, make_case, make_config, oracle_from_case


def test_library_exports_every_declared_symbol(built_lib):
    from shine_mapping_b200 import _abi
    header = open(os.path.join(ROOT, "include", "shine_b200.h")).read()
    declared = set(re.findall(r"\b(shine_[a-z0-9_]+)\s*\(", header))
    assert declared == set(_abi.SYMBOLS), declared ^ set(_abi.SYMBOLS)
    for name in declared:
        assert getattr(built_lib, name) is not None
    # 5: one shine_sdf_fwd / _step / _eikonal_step for every point-wise loss, chosen by flag (4 had one call per loss)
    assert built_lib.shine_abi_version() == _abi.ABI_VERSION == 5
    assert built_lib.shine_error_string(-2).decode().startswith("shine_b200: unsupported")


def test_struct_layouts_match_header():
    import ctypes as C
    from shine_mapping_b200 import _abi
    assert C.sizeof(_abi.ShineLevel) == 48
    assert C.sizeof(_abi.ShineOctree) == 16 + 8 * 48
    assert C.sizeof(_abi.ShineDecoder) == 12 * 8 + 16
    assert C.sizeof(_abi.ShineAdamTensor) == 48
    assert C.sizeof(_abi.ShineBoundaryInverse) == 8 * 8 + 8 * 4 + 8 * 8      # row_of_slot | slots | holders (SHINE_MAX_LEVELS = 8)
    assert C.sizeof(_abi.ShineBuildLevel) == 6 * 8 + 4 * 4 + 4 * 4
    assert C.sizeof(_abi.ShineBuild) == 8 + 6 * 8 + 8 * C.sizeof(_abi.ShineBuildLevel)


def test_abi_argument_checks_need_no_gpu(built_lib):
    import ctypes as C
    from shine_mapping_b200 import _abi
    d = _abi.ShineOctree()
    assert built_lib.shine_query_fwd(C.byref(d), None, 4, None, None) == -1          # num_levels == 0
    d.num_levels, d.feature_dim = 1, 6
    assert built_lib.shine_query_fwd(C.byref(d), None, 4, None, None) == -2          # F not a multiple of 4
    assert built_lib.shine_hash_insert(None, 16, None, None, 0, 0, None, None) == -1
    assert built_lib.shine_points_to_morton(None, 0, 12, None, None) == 0            # empty is fine
    # the octree build accepts world levels up to 15 (kaolin's int16 points); the checks run before any launch, so an
    # empty scan with placeholder pointers returns OK
    scratch = (C.c_int64 * 64)()
    plan = _abi.ShineBuild()
    plan.num_levels, plan.max_level = 1, 15
    plan.new_node_count = plan.new_corner_count = plan.new_corner_total = plan.new_node_total = C.addressof(scratch)
    plan.new_node_keys = plan.new_corner_keys = C.addressof(scratch)
    plan.lv[0].level, plan.lv[0].frame_node_set, plan.lv[0].frame_node_set_capacity = 15, C.addressof(scratch), 16
    assert built_lib.shine_octree_frame_nodes(C.byref(plan), None, 0, None) == 0
    assert built_lib.shine_octree_frame_corners(C.byref(plan), 0, None) == 0
    plan.max_level = plan.lv[0].level = 16
    assert built_lib.shine_octree_frame_nodes(C.byref(plan), None, 0, None) == -1
    assert built_lib.shine_octree_frame_corners(C.byref(plan), 0, None) == -1
    assert built_lib.shine_octree_assign_rows(C.byref(plan), None, 0, None) == -1
    assert built_lib.shine_octree_fill_nodes(C.byref(plan), None, 0, None, None) == -1
    plan.max_level = plan.lv[0].level = 15
    plan.new_node_total = None
    assert built_lib.shine_octree_frame_nodes(C.byref(plan), None, 0, None) == -1


def test_sdf_bce_calls_reject_unknown_flag_bits(built_lib):
    """A flag bit outside REDUCTION_SUM | WEIGHTED | TF32X1 | MORTON_ORDERED is SHINE_ERR_UNSUPPORTED, checked before
    anything else: a caller still setting bit 8, which ABI version 3 defined, gets an error, not another kernel.
    shine_sdf_fwd / shine_sdf_step run sdf_bce here (no loss bit)."""
    import ctypes as C
    from shine_mapping_b200 import _abi
    oct_, dec = C.byref(_abi.ShineOctree()), C.byref(_abi.ShineDecoder())      # num_levels == 0: an invalid octree
    calls = {
        "shine_sdf_infer": lambda f: built_lib.shine_sdf_infer(oct_, dec, None, 0, None, None, 0, f, None),
        "shine_sdf_bce_fwd": lambda f: built_lib.shine_sdf_bce_fwd(oct_, dec, None, None, None, 0, 1.0, 1.0, None, None,
                                                                   f, None),
        "shine_sdf_fwd": lambda f: built_lib.shine_sdf_fwd(oct_, dec, None, None, None, 0, 1.0, 1.0, 1.0, None, None, f,
                                                           None),
        "shine_sdf_step": lambda f: built_lib.shine_sdf_step(oct_, dec, None, None, None, 0, 1.0, 1.0, 1.0, None, None,
                                                             None, f, None),
    }
    known = _abi.FLAG_REDUCTION_SUM | _abi.FLAG_WEIGHTED | _abi.FLAG_TF32X1 | _abi.FLAG_MORTON_ORDERED
    for name, call in calls.items():
        assert call(known) == -1, name
        for flag in (8, 1 << 31):
            assert call(flag) == -2, (name, flag)


@pytest.mark.parametrize("name", GOLDEN_NAMES)
def test_update_reproduces_reference_tables(name):
    """FeatureOctree.update (vectorised) must give the reference's row counts and, via the oracle replay, the same
    node -> corner-row tables, including the append-only numbering of a second frame."""
    from shine_mapping_b200 import FeatureOctree
    case, exp = load_golden(name)
    c = case["cfg"]
    cfg = make_config(c["tree_level_feat"], c["tree_level_world"], c["leaf_vox_size"], device="cpu")
    octree = FeatureOctree(cfg)
    for fr in case["frames"]:
        octree.update(torch.from_numpy(fr))
    assert [tuple(p.shape) for p in octree.hier_features] == [t.shape for t in case["tables"]]
    oracle, _ = oracle_from_case(case)
    for lvl in range(c["tree_level_world"] + 1):
        assert octree.nodes_lookup_tables[lvl] == oracle.nodes_lookup_tables[lvl]
        assert octree.corners_lookup_tables[lvl] == oracle.corners_lookup_tables[lvl]
    for p in octree.hier_features:
        assert torch.equal(p[-1], torch.zeros(c["feature_dim"]))      # trash-bin row
    # every miss / hit recorded by the reference is consistent with the tables
    coord = torch.from_numpy(case["coord"])
    from shine_mapping_b200.feature_octree import points_to_morton, quantize_points
    for i, want in enumerate(exp["indices"]):
        level = c["tree_level_world"] - i
        keys = points_to_morton(quantize_points(coord, level)).tolist()
        table = octree.nodes_lookup_tables[level]
        got = np.array([table.get(k, [-1] * 8) for k in keys])
        assert np.array_equal(got, want)


def test_same_seed_same_feature_init_as_reference_call_order():
    """update() draws features with the reference's randn call shapes/order (feature_octree.py:139,153)."""
    from shine_mapping_b200 import FeatureOctree
    from oracle import shine_oracle as orc
    case = make_case(n_points=800, n_batch=10, feat_levels=3, seed=2, n_frames=2)
    cfg = make_config(3, device="cpu")
    torch.manual_seed(123)
    a = FeatureOctree(cfg)
    for fr in case["frames"]:
        a.update(torch.from_numpy(fr))
    torch.manual_seed(123)
    b = orc.OracleOctree(12, 3)
    for fr in case["frames"]:
        b.update(torch.from_numpy(fr))
    for p, q in zip(a.hier_features, b.hier_features):
        assert torch.equal(p.detach(), q.detach())


def test_constructor_contract_and_attributes():
    from shine_mapping_b200 import FeatureOctree
    cfg = make_config(4, device="cpu")
    o = FeatureOctree(cfg)
    assert (o.max_level, o.featured_level_num, o.free_level_num, o.feature_dim) == (12, 4, 9, 8)
    assert o.is_empty() and len(o.nodes_lookup_tables) == 13 and len(o.corners_lookup_tables) == 13
    cfg.tree_level_feat = 0
    with pytest.raises(ValueError, match="No level with grid features"):
        FeatureOctree(cfg)
    cfg.tree_level_feat = 4
    for world in (15, 16):
        cfg.tree_level_world = world
        if world == 15:
            assert FeatureOctree(cfg).max_level == 15
        else:
            with pytest.raises(ValueError, match="int16"):
                FeatureOctree(cfg)


def test_octree_pickles_like_the_reference_checkpoint():
    """save_checkpoint pickles the whole module (reference utils/tools.py:200-213)."""
    from shine_mapping_b200 import FeatureOctree
    case = make_case(n_points=600, n_batch=10, feat_levels=2, seed=4)
    o = FeatureOctree(make_config(2, device="cpu"))
    o.update(torch.from_numpy(case["frames"][0]))
    clone = pickle.loads(pickle.dumps(o))
    assert [tuple(p.shape) for p in clone.hier_features] == [tuple(p.shape) for p in o.hier_features]
    assert clone.nodes_lookup_tables[12] == o.nodes_lookup_tables[12]
    assert torch.equal(clone.hier_features[0], o.hier_features[0])


def test_module_to_moves_the_whole_structure():
    """`.to()` must carry the index arrays along with hier_features (checkpoints loaded with map_location)."""
    from shine_mapping_b200 import FeatureOctree
    case = make_case(n_points=600, n_batch=10, feat_levels=2, seed=4)
    o = FeatureOctree(make_config(2, device="cpu"))
    o.update(torch.from_numpy(case["frames"][0]))
    before = o.nodes_lookup_tables[12]
    o2 = o.to(torch.float32).cpu()          # dtype/device fns pass through integer arrays unchanged
    assert o2 is o and o.nodes_lookup_tables[12] == before
    assert o._levels[12].node_keys.dtype == torch.int64 and o._levels[12].node_ids.dtype == torch.int32
    o.update(torch.from_numpy(case["frames"][0]) + 0.01)     # still consistent after the move
    assert len(o.nodes_lookup_tables[12]) >= len(before)


def test_query_on_cpu_fails_loudly_no_fallback():
    from shine_mapping_b200 import Decoder, FeatureOctree, _abi, sdf_bce_step
    case = make_case(n_points=600, n_batch=10, feat_levels=2, seed=4)
    cfg = make_config(2, device="cpu")
    o, d = FeatureOctree(cfg), Decoder(cfg)
    o.update(torch.from_numpy(case["frames"][0]))
    with pytest.raises(_abi.ShineB200Error, match="no CPU fallback"):
        o.query_feature(torch.zeros(4, 3))
    with pytest.raises(_abi.ShineB200Error, match="no CPU fallback"):
        sdf_bce_step(o, d, torch.zeros(4, 3), torch.zeros(4), 0.01)


def test_decoder_surface_and_pretrained_state_dict_keys():
    """Module tree / state-dict keys / (out,in) layout of reference model/decoder.py:29-37."""
    from shine_mapping_b200 import Decoder
    from oracle import shine_oracle as orc
    cfg = make_config(2, device="cpu")
    d = Decoder(cfg)
    assert list(d.state_dict().keys()) == ["layers.0.weight", "layers.0.bias", "layers.1.weight", "layers.1.bias",
                                           "lout.weight", "lout.bias", "nclass_out.weight", "nclass_out.bias"]
    assert [tuple(v.shape) for v in d.state_dict().values()] == [(32, 8), (32,), (32, 32), (32,), (1, 32), (1,),
                                                                  (21, 32), (21,)]
    case, _ = load_golden("ref_c2_l4_pretrained_frozen")   # carries pretrained/geo_decoder_8dim.pth weights
    sd = d.state_dict()
    for k, v in case["dec"].items():
        sd[k] = torch.from_numpy(v)
    d.load_state_dict(sd)
    x = torch.randn(5, 8)
    params = {k: torch.from_numpy(v) for k, v in case["dec"].items()}
    assert torch.allclose(d.sdf(x), orc.decoder_sdf(x, params), atol=1e-6)
    assert d.fused_supported() and d.occupancy(x).shape == (5,) and d.sem_label(x).shape == (5,)
    for child in d.children():          # reference freeze_model (utils/tools.py:188-191)
        for p in child.parameters():
            p.requires_grad = False
    assert not any(p.requires_grad for p in d.parameters())


def test_config_loads_reference_schema_yaml(tmp_path):
    from shine_mapping_b200 import SHINEConfig
    y = tmp_path / "kitti_like.yaml"
    y.write_text("""
setting: {name: "t", output_root: "./e", pc_path: "p", pose_path: "q", calib_path: "c", load_model: False,
          model_path: "", first_frame_ref: False, begin_frame: 0, end_frame: 10, every_frame: 1, device: "cuda", gpu_id: "0"}
process: {min_range_m: 3.0, pc_radius_m: 50.0, min_z_m: -3.5, rand_downsample: False, vox_down_m: 0.05, rand_down_r: 0.2}
sampler: {surface_sample_range_m: 0.3, surface_sample_n: 3, free_sample_begin_ratio: 0.3, free_sample_end_dist_m: 0.8, free_sample_n: 3}
octree: {leaf_vox_size: 0.3, tree_level_world: 12, tree_level_feat: 3, feature_dim: 8, poly_int_on: True, octree_from_surface_samples: True}
decoder: {mlp_level: 2, mlp_hidden_dim: 32, freeze_after_frame: 0}
loss: {ray_loss: False, main_loss_type: sdf_bce, sigma_sigmoid_m: 0.1, loss_weight_on: False, behind_dropoff_on: False, ekional_loss_on: True, weight_e: 0.1}
continual: {continual_learning_reg: False, lambda_forget: 0, window_replay_on: False, window_radius_m: 0}
optimizer: {iters: 40000, batch_size: 4096, learning_rate: 0.05, weight_decay: 1e-7}
eval: {wandb_vis_on: False, o3d_vis_on: True, vis_freq_iters: 10000, save_freq_iters: 10000, mesh_freq_frame: 1, mc_res_m: 0.1,
       mc_with_octree: True, mc_local: False, mc_vis_level: 1, save_map: False, some_future_key: 1}
""")
    c = SHINEConfig()
    c.load(str(y))
    assert (c.tree_level_world, c.tree_level_feat, c.bs, c.lr, c.weight_decay) == (12, 3, 4096, 0.05, 1e-7)
    assert abs(c.scale - 1.0 / (0.3 * 2 ** 11)) < 1e-12 and c.infer_bs == 4096 * 16 and c.mc_query_level == 10
    assert c.window_radius == 100.0 and c.ekional_loss_on is True
    assert abs(c.sigma_sigmoid - 0.55 * 0.1 * c.scale) < 1e-15
    with pytest.raises(AttributeError):
        SHINEConfig(not_a_field=1)


def test_synth_sampler_contract():
    """Output contract of dataSampler.sample (utils/data_sampler.py:18-139) that the hot path consumes."""
    from shine_mapping_b200 import synth
    cfg = make_config(2, device="cpu")
    dirs = synth.lidar_directions(64)
    hits = synth.raycast_scene(torch.zeros(3), dirs, synth.default_boxes(), 3.0, 30.0)
    assert hits.shape[0] > 1000
    r = torch.linalg.norm(hits, dim=1)
    assert r.min() >= 3.0 - 1e-4 and r.max() <= 30.0 + 1e-4
    coord, label, weight = synth.sample_rays(hits * cfg.scale, torch.zeros(3), cfg, torch.Generator().manual_seed(0))
    m = hits.shape[0] * 6
    assert coord.shape == (m, 3) and label.shape == (m,) and weight.shape == (m,)
    w = weight.reshape(-1, 6)
    assert (w[:, :3] == 1).all() and (w[:, 3:] == -1).all()                     # ray-wise: 3 surface then 3 free
    assert label.reshape(-1, 6)[:, :3].abs().max() <= 0.3 * cfg.scale + 1e-9    # +-surface_sample_range, scaled
    assert coord.abs().max() <= 1.0
    # label is the signed displacement along the ray: |coord - hit| == |label|
    disp = torch.linalg.norm(coord.reshape(-1, 6, 3) - (hits * cfg.scale).unsqueeze(1), dim=2)
    assert torch.allclose(disp, label.reshape(-1, 6).abs(), atol=2e-7)


def test_sample_pool_morton_order_keeps_the_sampler_and_orders_the_batch():
    """SamplePool.sort_morton(): same samples, Z-order; get_batch() then draws the same randint index stream as before and
    hands the samples out in ascending index = Morton order (a subsequence of a Morton-ordered sequence is Morton-ordered);
    ordered=False gives the order drawn; an unsorted pool refuses ordered=True."""
    from shine_mapping_b200 import synth
    from shine_mapping_b200.feature_octree import points_to_morton, quantize_points
    g = torch.Generator().manual_seed(3)
    pool = synth.SamplePool("cpu")
    coord = torch.rand(5000, 3, generator=g) * 1.6 - 0.8
    pool.append(coord, torch.arange(5000, dtype=torch.float32), torch.ones(5000))
    with pytest.raises(ValueError):
        pool.get_batch(10, ordered=True)
    assert pool.ordered is False
    pool.sort_morton()
    assert pool.ordered and len(pool) == 5000
    keys = points_to_morton(quantize_points(pool.coord_pool, 16))
    assert bool((keys[1:] >= keys[:-1]).all())
    assert torch.equal(torch.sort(pool.sdf_label_pool).values, torch.arange(5000, dtype=torch.float32))   # a permutation
    assert torch.equal(pool.coord_pool, coord[pool.sdf_label_pool.long()])                                 # rows moved together
    c, l, w = pool.get_batch(700, torch.Generator().manual_seed(9))
    bk = points_to_morton(quantize_points(c, 16))
    assert bool((bk[1:] >= bk[:-1]).all())
    for lvl in (12, 9):          # ordered at every coarser level too (Morton prefixes)
        ck = points_to_morton(quantize_points(c, lvl))
        assert bool((ck[1:] >= ck[:-1]).all())
    c2, l2, _ = pool.get_batch(700, torch.Generator().manual_seed(9), ordered=False)
    assert torch.equal(torch.sort(l).values, torch.sort(l2).values)          # the same index multiset, another order
    assert not torch.equal(l, l2)
    pool.append(coord[:3], torch.zeros(3), torch.ones(3))
    assert pool.ordered is False                                              # appending breaks the order until re-sorted


def test_free_space_samples_go_last_and_sees_a_node_matches_the_node_tables():
    """FeatureOctree.sees_a_node == membership in the coarsest featured level's node dict (every leaf has its ancestors);
    SamplePool.sort_morton(octree=...) puts the samples without any node behind the others, both parts in Z-order, and a
    batch inherits that layout."""
    from shine_mapping_b200 import FeatureOctree, synth
    from shine_mapping_b200.feature_octree import points_to_morton, quantize_points
    case = make_case(n_points=2500, n_batch=4000, feat_levels=3, seed=17)
    cfg = make_config(3, device="cpu")
    octree = FeatureOctree(cfg)
    for fr in case["frames"]:
        octree.update(torch.from_numpy(np.asarray(fr)))
    coord = torch.from_numpy(case["coord"])
    seen = octree.sees_a_node(coord)
    lvl = octree.free_level_num
    table = octree.nodes_lookup_tables[lvl]
    keys = points_to_morton(quantize_points(coord, lvl)).tolist()
    assert seen.tolist() == [k in table for k in keys]
    finer = octree.nodes_lookup_tables[octree.max_level]
    leaf_keys = points_to_morton(quantize_points(coord, octree.max_level)).tolist()
    assert all(s for s, k in zip(seen.tolist(), leaf_keys) if k in finer)       # a leaf hit implies a coarse hit
    assert 0 < int(seen.sum()) < len(seen)
    pool = synth.SamplePool("cpu")
    pool.append(coord, torch.from_numpy(case["label"]), torch.from_numpy(case["weight"]))
    pool.sort_morton(octree=octree)
    s2 = octree.sees_a_node(pool.coord_pool)
    n_near = int(s2.sum())
    assert bool(s2[:n_near].all()) and not bool(s2[n_near:].any())
    for part in (pool.coord_pool[:n_near], pool.coord_pool[n_near:]):
        k = points_to_morton(quantize_points(part, 16))
        assert bool((k[1:] >= k[:-1]).all())
    c, _, _ = pool.get_batch(1000, torch.Generator().manual_seed(2))
    sb = octree.sees_a_node(c)
    nb = int(sb.sum())
    assert bool(sb[:nb].all()) and not bool(sb[nb:].any())
