"""`FeatureOctree` — drop-in for reference model/feature_octree.py:29-298 whose queries run as sm_90a kernels.

Same constructor, attributes and methods as the reference class (SURVEY.md §8b).  What changes underneath:

* the per-level Python dicts `nodes_lookup_tables[level]` (Morton -> 8 corner rows) become device hash tables
  of 64-byte slots probed inside the kernels (`csrc/shine_b200.cu`); the dict views are still available
  (built lazily from the authoritative arrays) for callers that read them;
* `update()` (reference :114-166) is vectorised torch code instead of Python dict loops but reproduces the
  reference's row numbering exactly (lexicographic `torch.unique(dim=0)` order, append-only) and draws the
  new features with the same `randn` calls, so tables match the reference under the same seed/device;
* `get_indices`, `query_feature` (+ its autograd backward) call the C ABI; there is no CPU path.
"""
from __future__ import annotations

import ctypes as C
import os

import torch
import torch.nn as nn

from . import _abi
from .config import SHINEConfig

# --------------------------------------------------------------------------------------------------------
# integer helpers (host logic of update(); the kernels carry their own device versions)
# --------------------------------------------------------------------------------------------------------


def quantize_points(x: torch.Tensor, level: int) -> torch.Tensor:
    """floor(clamp(2^level (x+1)/2, 0, 2^level-1)) in fp32 -> int64 xyz (kaolin quantize_points semantics,
    reference call site model/feature_octree.py:203)."""
    res = float(2 ** level)
    return torch.floor(torch.clamp(res * (x.float() + 1.0) / 2.0, 0, res - 1.0)).long()


def _spread3(v: torch.Tensor) -> torch.Tensor:
    v = v & 0xFFFF
    v = (v | (v << 16)) & 0x0000FF0000FF
    v = (v | (v << 8)) & 0x00F00F00F00F
    v = (v | (v << 4)) & 0x0C30C30C30C3
    v = (v | (v << 2)) & 0x249249249249
    return v


def _compact3(v: torch.Tensor) -> torch.Tensor:
    v = v & 0x249249249249
    v = (v | (v >> 2)) & 0x0C30C30C30C3
    v = (v | (v >> 4)) & 0x00F00F00F00F
    v = (v | (v >> 8)) & 0x0000FF0000FF
    v = (v | (v >> 16)) & 0xFFFF
    return v


def points_to_morton(p: torch.Tensor) -> torch.Tensor:
    """x -> bit 3i+2, y -> 3i+1, z -> 3i (kaolin points_to_morton, call site model/feature_octree.py:204)."""
    p = p.long()
    return (_spread3(p[..., 0]) << 2) | (_spread3(p[..., 1]) << 1) | _spread3(p[..., 2])


def morton_to_points(m: torch.Tensor) -> torch.Tensor:
    m = m.long()
    return torch.stack((_compact3(m >> 2), _compact3(m >> 1), _compact3(m)), dim=-1)


_CORNER_OFFSETS = [[(i >> 2) & 1, (i >> 1) & 1, i & 1] for i in range(8)]


def points_to_corners(p: torch.Tensor) -> torch.Tensor:
    """corner i = p + ((i>>2)&1, (i>>1)&1, i&1): the order pinned by model/feature_octree.py:186-195."""
    off = torch.tensor(_CORNER_OFFSETS, dtype=p.dtype, device=p.device)
    return p.unsqueeze(-2) + off


def _lex_key(c: torch.Tensor) -> torch.Tensor:
    """Order-preserving key of lexicographic (x, y, z) — the order of torch.unique(dim=0) (reference :132) on kaolin's
    int16 corner points, where the coordinate 2^15 of the + face at world level 15 wraps to -2^15 and comes first:
    c ^ 0x8000 maps that order onto unsigned 16-bit order (csrc/shine_octree_build.cu keys its corners the same way)."""
    c = c.long() ^ 0x8000
    return (c[..., 0] << 32) | (c[..., 1] << 16) | c[..., 2]


def _lex_to_points(k: torch.Tensor) -> torch.Tensor:
    return torch.stack((k >> 32, (k >> 16) & 0xFFFF, k & 0xFFFF), -1) ^ 0x8000


# kaolin's octree points are int16: level 15 is the deepest whose corner coordinates (0 .. 2^15) fit 16 bits
MAX_WORLD_LEVEL = 15


def _next_pow2(n: int) -> int:
    return 1 << max(4, (int(n) - 1).bit_length())


class _LevelState:
    """Authoritative per-level arrays (world level numbering)."""

    def __init__(self, device):
        self.node_keys = torch.empty(0, dtype=torch.int64, device=device)        # insertion order (Morton per frame)
        self.node_ids = torch.empty(0, 8, dtype=torch.int32, device=device)      # rows of the 8 corners
        self.node_keys_sorted = torch.empty(0, dtype=torch.int64, device=device)
        self.corner_lex_sorted = torch.empty(0, dtype=torch.int64, device=device)
        self.corner_rows_sorted = torch.empty(0, dtype=torch.int64, device=device)
        self.corner_morton_by_row = torch.empty(0, dtype=torch.int64, device=device)
        self.hash = None          # uint8 [capacity * 64] device tensor
        self.hash_capacity = 0
        self.hash_count = 0       # nodes already inserted
        self.corner_hash = None   # int64 [capacity * 2] device tensor (16-byte slots {lexicographic key, row}), CUDA build
        self.corner_hash_capacity = 0
        self.corner_hash_count = 0


# --------------------------------------------------------------------------------------------------------
# autograd bridge for query_feature
# --------------------------------------------------------------------------------------------------------


class _QueryCoordGrad(torch.autograd.Function):
    """G[p,a] = sum_levels sum_c dw_c/da <f_c, dfeat_p>: the backward of query_feature w.r.t. the coordinates, itself
    differentiable w.r.t. dfeat and the tables (what `autograd.grad(pred, coord, create_graph=True)` needs for the
    eikonal / normal losses, reference utils/tools.py:175-185)."""

    @staticmethod
    def forward(ctx, octree, coord, dfeat, *tables):
        n = coord.shape[0]
        dfeat = dfeat.contiguous()
        out = torch.empty(n, 3, dtype=torch.float32, device=coord.device)
        desc = octree._descriptor(tables, None)
        _abi.check(_abi.lib().shine_query_coord_grad(C.byref(desc), _abi.ptr(coord), n, _abi.ptr(dfeat), _abi.ptr(out),
                                                     _abi.stream_ptr(coord.device)), "shine_query_coord_grad")
        ctx.octree = octree
        ctx.save_for_backward(coord, dfeat, *tables)
        return out

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, dG):
        coord, dfeat, *tables = ctx.saved_tensors
        octree = ctx.octree
        n = coord.shape[0]
        dG = dG.contiguous()
        lib, stream = _abi.lib(), _abi.stream_ptr(coord.device)
        d_dfeat = None
        if ctx.needs_input_grad[2]:
            d_dfeat = torch.empty_like(dfeat)
            desc = octree._descriptor(tables, None)
            _abi.check(lib.shine_query_tangent_fwd(C.byref(desc), _abi.ptr(coord), n, _abi.ptr(dG), _abi.ptr(d_dfeat),
                                                   stream), "shine_query_tangent_fwd")
        grads = [None] * len(tables)
        if any(ctx.needs_input_grad[3:]):
            full = [torch.zeros_like(t) for t in tables]
            desc = octree._descriptor(tables, full)
            _abi.check(lib.shine_query_tangent_bwd(C.byref(desc), _abi.ptr(coord), n, _abi.ptr(dG), _abi.ptr(dfeat),
                                                   stream), "shine_query_tangent_bwd")
            grads = [g if need else None for g, need in zip(full, ctx.needs_input_grad[3:])]
        return (None, None, d_dfeat, *grads)


class _QueryFeature(torch.autograd.Function):
    """query_feature forward = shine_query_fwd, backward = shine_query_bwd (dense grads like the reference's
    index_put_(accumulate=True), but scatter-added with vector atomics and misses skipped); the gradient w.r.t. the
    coordinates is `_QueryCoordGrad`, which supports a second backward."""

    @staticmethod
    def forward(ctx, octree, coord, *tables):
        n = coord.shape[0]
        out = torch.empty(n, octree.feature_dim, dtype=torch.float32, device=coord.device)
        desc = octree._descriptor(tables, None)
        _abi.check(_abi.lib().shine_query_fwd(C.byref(desc), _abi.ptr(coord), n, _abi.ptr(out),
                                              _abi.stream_ptr(coord.device)), "shine_query_fwd")
        ctx.octree = octree
        ctx.save_for_backward(coord, *tables)
        return out

    @staticmethod
    def backward(ctx, dfeat):
        coord, *tables = ctx.saved_tensors
        octree = ctx.octree
        grads = [None] * len(tables)
        if any(ctx.needs_input_grad[2:]):
            with torch.no_grad():
                full = [torch.zeros_like(t) for t in tables]
                desc = octree._descriptor(tables, full, n_points=coord.shape[0])
                d = dfeat.detach().contiguous()
                _abi.check(_abi.lib().shine_query_bwd(C.byref(desc), _abi.ptr(coord), coord.shape[0], _abi.ptr(d),
                                                      _abi.stream_ptr(coord.device)), "shine_query_bwd")
                octree._reduce_replicas(desc, coord.device)
            grads = [g if need else None for g, need in zip(full, ctx.needs_input_grad[2:])]
        dcoord = None
        if ctx.needs_input_grad[1]:
            dcoord = _QueryCoordGrad.apply(octree, coord.detach(), dfeat, *tables)
        return (None, dcoord, *grads)


# --------------------------------------------------------------------------------------------------------
# FeatureOctree
# --------------------------------------------------------------------------------------------------------


class FeatureOctree(nn.Module):

    def __init__(self, config: SHINEConfig):
        super().__init__()
        # [0 .. max_level]; level 0 is the root (reference :35-44)
        self.max_level = config.tree_level_world
        self.leaf_vox_size = config.leaf_vox_size
        self.featured_level_num = config.tree_level_feat
        self.free_level_num = self.max_level - self.featured_level_num + 1
        self.feature_dim = config.feature_dim
        self.feature_std = config.feature_std
        self.polynomial_interpolation = config.poly_int_on
        self.device = config.device
        if self.featured_level_num < 1:
            raise ValueError('No level with grid features!')
        if self.featured_level_num > _abi.MAX_LEVELS:
            raise ValueError(f'tree_level_feat > {_abi.MAX_LEVELS} is not supported by the sm_90a kernels')
        if self.max_level > MAX_WORLD_LEVEL:
            raise ValueError(f'tree_level_world > {MAX_WORLD_LEVEL} is not supported: kaolin keeps octree points as int16, '
                             f'so the corners of level {MAX_WORLD_LEVEL + 1} (coordinates up to 2^{MAX_WORLD_LEVEL + 1}) '
                             'cannot be represented')
        self._levels = [_LevelState(self.device) for _ in range(self.max_level + 1)]
        self._dict_cache = None
        self._desc_cache = {}
        self._grad_scratch = {}   # k -> zero-invariant replica scratch (gradient privatisation)
        # coarse -> fine; the last row of each table is the trash-bin (reference :61-63)
        self.hier_features = nn.ParameterList([])
        self._last_coord = None
        self._hier_idx = []
        # incremental mapping state (reference :70-72)
        self.importance_weight = []
        self.features_last_frame = []
        self.to(config.device)

    # ---- dict views kept for callers that read the reference's tables (reference :46-52) -------------------

    def _build_dicts(self):
        if self._dict_cache is None:
            corners, nodes = [], []
            for st in self._levels:
                cm = st.corner_morton_by_row.tolist()
                corners.append(dict(zip(cm, range(len(cm)))))
                nodes.append(dict(zip(st.node_keys.tolist(), st.node_ids.tolist())))
            self._dict_cache = (corners, nodes)
        return self._dict_cache

    @classmethod
    def from_lookup_tables(cls, config: SHINEConfig, corners, nodes, hier_features, importance_weight=(),
                           features_last_frame=()):
        """The inverse of `_build_dicts`: an octree on `config.device` from the reference's tables (model/feature_octree.py
        :46-72) — per world level 0..tree_level_world a dict Morton -> row (`corners`) and a dict Morton -> 8 rows
        (`nodes`), and the feature tables coarse -> fine with their trailing trash row.  Node order is the dicts'
        insertion order, so the dict views, `get_indices`, the fused kernels and a later `update()` behave as if the map
        had been grown here.  The tables come from a file: what the kernels would index with is checked, and a
        violation is a ValueError naming the table."""
        self = cls(config)
        dev = self.device
        if len(corners) != self.max_level + 1 or len(nodes) != self.max_level + 1:
            raise ValueError(f"corners_lookup_tables / nodes_lookup_tables: {len(corners)} / {len(nodes)} levels, "
                             f"tree_level_world {self.max_level} needs {self.max_level + 1}")
        tables = [torch.as_tensor(t).detach() for t in hier_features]
        if len(tables) not in (0, self.featured_level_num):
            raise ValueError(f"hier_features: {len(tables)} tables, tree_level_feat is {self.featured_level_num}")
        for t in tables:
            self.hier_features.append(nn.Parameter(t.to(dev).clone().contiguous()))
        for lvl, st in enumerate(self._levels):
            what = f"level {lvl}"
            cm = torch.tensor(list(corners[lvl].keys()), dtype=torch.int64).reshape(-1)
            cr = torch.tensor(list(corners[lvl].values()), dtype=torch.int64).reshape(-1)
            if not torch.equal(torch.sort(cr).values, torch.arange(cr.numel())):
                raise ValueError(f"corners_lookup_tables {what}: the rows are not a numbering 0 .. {cr.numel() - 1}")
            try:
                nk = torch.tensor(list(nodes[lvl].keys()), dtype=torch.int64).reshape(-1)
                ni = torch.tensor(list(nodes[lvl].values()), dtype=torch.int64).reshape(nk.numel(), 8)
            except (ValueError, RuntimeError, TypeError):
                raise ValueError(f"nodes_lookup_tables {what}: every node holds 8 corner rows") from None
            if ni.numel() and (int(ni.min()) < -2 ** 31 or int(ni.max()) >= 2 ** 31):
                raise ValueError(f"nodes_lookup_tables {what}: corner row outside int32")
            st.node_keys = nk.to(dev)
            st.node_ids = ni.to(torch.int32).to(dev)
            by_row = torch.empty(cr.numel(), dtype=torch.int64)
            by_row[cr] = cm
            st.corner_morton_by_row = by_row.to(dev)
            self._refresh_sorted(st)
        self.check_tables()
        for name, given in (("importance_weight", importance_weight), ("features_last_frame", features_last_frame)):
            given = [torch.as_tensor(t).detach() for t in given]
            if given and [tuple(t.shape) for t in given] != [tuple(p.shape) for p in self.hier_features]:
                raise ValueError(f"{name}: shapes {[tuple(t.shape) for t in given]} do not match hier_features")
            setattr(self, name, [t.to(dev).float().clone() for t in given])
        return self

    def check_tables(self) -> None:
        """Consistency of the per-level arrays with the feature tables, for a map that arrives from a file: the kernels
        index the tables with the stored corner rows.  A violation is a ValueError naming the table, not a fault in a
        kernel.  A stored row is never -1 (what a miss yields) nor the trash row."""
        if len(self.hier_features) not in (0, self.featured_level_num):
            raise ValueError(f"hier_features: {len(self.hier_features)} tables, tree_level_feat is {self.featured_level_num}")
        for lvl, st in enumerate(self._levels):
            what = f"level {lvl}"
            k = lvl - self.free_level_num
            if k < 0 or not len(self.hier_features):
                if st.node_keys.numel() or st.corner_morton_by_row.numel():
                    raise ValueError(f"corners_lookup_tables / nodes_lookup_tables {what}: entries at a level without features")
                continue
            t = self.hier_features[k]
            if t.dim() != 2 or t.shape[0] < 1 or t.shape[1] != self.feature_dim or t.dtype != torch.float32:
                raise ValueError(f"hier_features[{k}]: {t.dtype} {tuple(t.shape)}, expected float32 [rows + 1, "
                                 f"{self.feature_dim}]")
            rows = t.shape[0] - 1
            if st.corner_morton_by_row.numel() != rows:
                raise ValueError(f"corners_lookup_tables {what}: {st.corner_morton_by_row.numel()} corners for {rows} "
                                 "feature rows (+ the trash row)")
            if st.node_keys.dim() != 1 or tuple(st.node_ids.shape) != (st.node_keys.numel(), 8):
                raise ValueError(f"nodes_lookup_tables {what}: every node holds 8 corner rows")
            if st.node_keys.numel():
                if int(st.node_keys.min()) < 0 or int(st.node_keys.max()) >= 8 ** lvl:
                    raise ValueError(f"nodes_lookup_tables {what}: Morton code outside the level")
                if int(st.node_ids.min()) < 0 or int(st.node_ids.max()) >= rows:
                    raise ValueError(f"nodes_lookup_tables {what}: corner row outside [0, {rows})")

    @property
    def corners_lookup_tables(self):
        return self._build_dicts()[0]

    @property
    def nodes_lookup_tables(self):
        return self._build_dicts()[1]

    @property
    def hierarchical_indices(self):
        """Bottom-up list of [N,8] int64 for the last queried batch (reference :66-67).  Materialised lazily:
        the fused kernels never need it, only `Mesher.query_points` / `cal_regularization` read it."""
        if not self._hier_idx and self._last_coord is not None:
            self._hier_idx = self._compute_indices(self._last_coord)
        return self._hier_idx

    @hierarchical_indices.setter
    def hierarchical_indices(self, value):
        self._hier_idx = value
        self._last_coord = None

    def __getstate__(self):
        state = self.__dict__.copy()
        state["_dict_cache"] = None
        state["_desc_cache"] = {}
        state["_grad_scratch"] = {}
        state["_last_coord"] = None
        state["_hier_idx"] = []
        state.pop("_touched_rows", None)   # incre_loop's device scratch (ctypes descriptors): rebuilt on demand
        levels = []
        for st in self._levels:  # device hash tables are rebuilt on demand after unpickling
            cp = _LevelState.__new__(_LevelState)
            cp.__dict__.update(st.__dict__)
            cp.hash, cp.hash_capacity, cp.hash_count = None, 0, 0
            cp.corner_hash, cp.corner_hash_capacity, cp.corner_hash_count = None, 0, 0
            levels.append(cp)
        state["_levels"] = levels
        return state

    def _apply(self, fn, *args, **kwargs):
        """`.to()/.cuda()/.cpu()`: move the per-level index arrays together with the parameters; device hash tables,
        replica scratch and cached descriptors are rebuilt on demand."""
        super()._apply(fn, *args, **kwargs)
        for st in self._levels:
            for name in ("node_keys", "node_ids", "node_keys_sorted", "corner_lex_sorted", "corner_rows_sorted",
                         "corner_morton_by_row"):
                setattr(st, name, fn(getattr(st, name)))
            st.hash, st.hash_capacity, st.hash_count = None, 0, 0
            st.corner_hash, st.corner_hash_capacity, st.corner_hash_count = None, 0, 0
        self.importance_weight = [fn(t) for t in self.importance_weight]
        self.features_last_frame = [fn(t) for t in self.features_last_frame]
        self._grad_scratch, self._desc_cache, self._last_coord, self._hier_idx = {}, {}, None, []
        if len(self.hier_features):
            self.device = self.hier_features[0].device
        return self

    # ---- reference API -------------------------------------------------------------------------------------

    def set_zero(self):
        """Re-zero the trash-bin rows (reference :78-81).  Written through `.data`: the reference does this with an
        untracked copy too (:80-81), so a second query before the first result is back-propagated must not trip
        autograd's saved-tensor version check (shine_batch.py:155-160 queries `coord_near` that way)."""
        for p in self.hier_features:
            p.data[-1].zero_()

    def forward(self, x):
        return self.query_feature(x)

    def get_morton(self, sample_points, level):
        points_morton = points_to_morton(quantize_points(sample_points, level))
        sample_points_with_morton = torch.hstack((sample_points, points_morton.view(-1, 1)))
        return sample_points_with_morton, set(points_morton.cpu().numpy())

    @torch.no_grad()
    def sees_a_node(self, coord: torch.Tensor) -> torch.Tensor:
        """bool [N]: does the point fall into a node of ANY featured level?  Every leaf node has all its ancestors
        (update() derives the coarser node sets from the leaf keys, reference :129-143), so this is a lookup at the
        coarsest featured level.  Plain torch (sorted keys + searchsorted) on whatever device the octree lives on: a
        set-up-time helper for the sample pool (`SamplePool.sort_morton(octree=...)`), not part of the step."""
        lvl = self.free_level_num
        keys = self._levels[lvl].node_keys
        if keys.numel() == 0:
            return torch.zeros(coord.shape[0], dtype=torch.bool, device=coord.device)
        table = torch.sort(keys.to(coord.device)).values
        q = points_to_morton(quantize_points(coord, lvl))
        pos = torch.searchsorted(table, q).clamp_(max=table.numel() - 1)
        return table[pos] == q

    def get_octree_nodes(self, level):
        """Node centres at `level` in the [-1,1] cube (reference :94-101)."""
        nodes = morton_to_points(self._levels[level].node_keys).cpu().numpy()
        node_size = 2 ** (1 - level)
        return (nodes * node_size) - 1.0 + 0.5 * node_size

    def is_empty(self):
        return len(self.hier_features) == 0

    def clear_temp(self):
        self._hier_idx = []
        self._last_coord = None
        self.importance_weight = []
        self.features_last_frame = []

    @torch.no_grad()
    def update(self, surface_points, incremental_on=False):
        """Grow the octree from new surface points (reference :114-166), vectorised.

        Per featured level i: occupied nodes = unique(leaf_morton >> 3(W-i)) in Morton order (what kaolin's
        unbatched_pointcloud_to_spc yields, reference :116-122); nodes not seen before are new (:124-128); their
        corners, made unique in lexicographic order (:131-132), get row ids — 0..n-1 for the first frame
        (:135-137), appended after the existing rows for later frames (:148-151); the trash row is re-appended
        last (:139-142,153-156); each new node stores its 8 corner rows (:162-166)."""
        dev = self.device
        pts = surface_points.to(dev)
        if pts.is_cuda:
            return self._update_cuda(pts.float().contiguous(), incremental_on)
        # CPU tensors: host-side restatement with torch ops (the query kernels refuse CPU tensors anyway; this path
        # exists so that table numbering can be checked against the oracle without a GPU)
        for st in self._levels:
            self._refresh_sorted(st)
        leaf = torch.unique(points_to_morton(quantize_points(pts, self.max_level)))
        for i in range(self.max_level + 1):
            if i < self.free_level_num:
                continue
            st = self._levels[i]
            nodes_m = torch.unique(leaf >> (3 * (self.max_level - i)))
            if st.node_keys_sorted.numel():
                pos = torch.searchsorted(st.node_keys_sorted, nodes_m).clamp_(max=st.node_keys_sorted.numel() - 1)
                is_new = st.node_keys_sorted[pos] != nodes_m
                new_m = nodes_m[is_new]
            else:
                new_m = nodes_m
            if new_m.numel() == 0:
                continue
            corners = points_to_corners(morton_to_points(new_m))            # [n, 8, 3]
            lex = _lex_key(corners).reshape(-1)
            lex_unique = torch.unique(lex)                                    # lexicographic (x, y, z)
            cur = i - self.free_level_num
            if st.corner_lex_sorted.numel() == 0:   # first frame of this level
                fresh = lex_unique
                pre_size = 0
                fts = self.feature_std * torch.randn(fresh.numel() + 1, self.feature_dim, device=dev)
                fts[-1] = 0.0
                self.hier_features.append(nn.Parameter(fts))
                if incremental_on:
                    self.importance_weight.append(torch.zeros(fresh.numel() + 1, self.feature_dim, device=dev))
                    self.features_last_frame.append(fts.clone())
            else:
                pos = torch.searchsorted(st.corner_lex_sorted, lex_unique).clamp_(max=st.corner_lex_sorted.numel() - 1)
                fresh = lex_unique[st.corner_lex_sorted[pos] != lex_unique]
                pre_size = st.corner_lex_sorted.numel()
                new_fts = self.feature_std * torch.randn(fresh.numel() + 1, self.feature_dim, device=dev)
                new_fts[-1] = 0.0
                self.hier_features[cur] = nn.Parameter(torch.cat((self.hier_features[cur].data[:-1], new_fts), 0))
                if incremental_on:
                    new_w = torch.zeros(fresh.numel() + 1, self.feature_dim, device=dev)
                    self.importance_weight[cur] = torch.cat((self.importance_weight[cur][:-1], new_w), 0)
                    self.features_last_frame[cur] = self.hier_features[cur].data.clone()
            if fresh.numel():
                fresh_rows = pre_size + torch.arange(fresh.numel(), device=dev)
                all_lex = torch.cat((st.corner_lex_sorted, fresh))
                all_rows = torch.cat((st.corner_rows_sorted, fresh_rows))
                order = torch.argsort(all_lex)
                st.corner_lex_sorted, st.corner_rows_sorted = all_lex[order], all_rows[order]
                st.corner_morton_by_row = torch.cat((st.corner_morton_by_row, points_to_morton(_lex_to_points(fresh))))
            ids = st.corner_rows_sorted[torch.searchsorted(st.corner_lex_sorted, lex)].reshape(-1, 8).to(torch.int32)
            st.node_keys = torch.cat((st.node_keys, new_m))
            st.node_ids = torch.cat((st.node_ids, ids))
            st.node_keys_sorted = torch.sort(torch.cat((st.node_keys_sorted, new_m))).values
        self._dict_cache = None
        self._desc_cache = {}
        self._hier_idx = []
        self._last_coord = None

    @staticmethod
    def _refresh_sorted(st):
        """The sorted search arrays of the torch path, rebuilt from the authoritative per-row / per-node arrays when the
        CUDA build path (which does not maintain them) grew the level."""
        if st.node_keys_sorted.numel() != st.node_keys.numel():
            st.node_keys_sorted = torch.sort(st.node_keys).values
        if st.corner_lex_sorted.numel() != st.corner_morton_by_row.numel():
            lex = _lex_key(morton_to_points(st.corner_morton_by_row))
            order = torch.argsort(lex)
            st.corner_lex_sorted, st.corner_rows_sorted = lex[order], order

    def _grow_features(self, cur: int, n_fresh: int, first: bool, incremental_on: bool, dev):
        """New rows of a level: feature_std * randn with the reference's call shapes (model/feature_octree.py:139,153),
        trash row re-appended last."""
        fts = self.feature_std * torch.randn(n_fresh + 1, self.feature_dim, device=dev)
        fts[-1] = 0.0
        if first:
            self.hier_features.append(nn.Parameter(fts))
            if incremental_on:
                self.importance_weight.append(torch.zeros(n_fresh + 1, self.feature_dim, device=dev))
                self.features_last_frame.append(fts.clone())
        else:
            self.hier_features[cur] = nn.Parameter(torch.cat((self.hier_features[cur].data[:-1], fts), 0))
            if incremental_on:
                new_w = torch.zeros(n_fresh + 1, self.feature_dim, device=dev)
                self.importance_weight[cur] = torch.cat((self.importance_weight[cur][:-1], new_w), 0)
                self.features_last_frame[cur] = self.hier_features[cur].data.clone()

    def _update_cuda(self, pts, incremental_on):
        """update() as kernels over the scan (csrc/shine_octree_build.cu): no unique/sort/searchsorted over the scan, one
        radix sort over the NEW nodes and corners only; two small count read-backs size the tables and the new feature
        rows."""
        lib = _abi.lib()
        dev = pts.device
        st_ptr = _abi.stream_ptr(dev)
        n = pts.shape[0]
        if n == 0:
            return
        L = self.featured_level_num
        levels = list(range(self.free_level_num, self.max_level + 1))         # coarse -> fine, like hier_features
        counts = torch.zeros(2 * L + 2, dtype=torch.int32, device=dev)
        plan = _abi.ShineBuild()
        plan.num_levels, plan.max_level = L, self.max_level
        plan.new_node_count = counts.data_ptr()
        plan.new_corner_count = counts.data_ptr() + 4 * L
        plan.new_corner_total = counts.data_ptr() + 8 * L
        plan.new_node_total = counts.data_ptr() + 8 * L + 4
        set_cap = _next_pow2(2 * n)
        node_sets = torch.full((L, set_cap), -1, dtype=torch.int64, device=dev)
        node_list = torch.empty(L * n, dtype=torch.int64, device=dev)
        plan.new_node_keys = node_list.data_ptr()
        for l, lvl in enumerate(levels):
            st = self._levels[lvl]
            self._ensure_level_tables(st, lvl)
            b = plan.lv[l]
            b.level, b.nodes_before, b.rows_before = lvl, int(st.node_keys.numel()), int(st.corner_morton_by_row.numel())
            b.node_slots = st.hash.data_ptr() if st.hash is not None else None
            b.node_capacity = st.hash_capacity
            b.frame_node_set, b.frame_node_set_capacity = node_sets[l].data_ptr(), set_cap
        _abi.check(lib.shine_octree_frame_nodes(C.byref(plan), _abi.ptr(pts), n, st_ptr), "shine_octree_frame_nodes")
        c_nodes = counts[:L].tolist()                                          # read-back 1
        n_new = sum(c_nodes)
        if n_new == 0:
            return
        keep = []       # scratch referenced by the plan must outlive the launches
        for l, lvl in enumerate(levels):
            st = self._levels[lvl]
            b = plan.lv[l]
            self._reserve_node_table(st, lvl, b.nodes_before + c_nodes[l])
            self._reserve_corner_table(st, b.rows_before + 8 * c_nodes[l])
            b.node_slots, b.node_capacity = st.hash.data_ptr(), st.hash_capacity
            b.corner_slots, b.corner_capacity = st.corner_hash.data_ptr(), st.corner_hash_capacity
            cap = _next_pow2(16 * max(c_nodes[l], 1))
            cs = torch.full((cap,), -1, dtype=torch.int64, device=dev)
            ids = torch.empty(max(c_nodes[l], 1), 8, dtype=torch.int32, device=dev)
            b.frame_corner_set, b.frame_corner_set_capacity = cs.data_ptr(), cap
            b.node_ids_out = ids.data_ptr()
            keep.append((cs, ids))
        # sort input: the node entries, then room for the corner entries frame_corners appends
        keys = torch.empty(9 * n_new, dtype=torch.int64, device=dev)
        keys[:n_new].copy_(node_list[:n_new])
        plan.new_corner_keys = keys.data_ptr() + 8 * n_new
        _abi.check(lib.shine_octree_frame_corners(C.byref(plan), n_new, st_ptr), "shine_octree_frame_corners")
        c_corners = counts[L:2 * L + 1].tolist()                               # read-back 2
        total = c_corners[-1]
        sorted_keys = torch.empty(total + n_new, dtype=torch.int64, device=dev)  # [corners | nodes]
        nbytes = int(lib.shine_octree_sort_scratch_bytes(total + n_new))
        scratch = torch.empty(max(nbytes, 16), dtype=torch.uint8, device=dev)
        _abi.check(lib.shine_octree_sort_new_keys(_abi.ptr(keys), _abi.ptr(sorted_keys), total + n_new, _abi.ptr(scratch),
                                                  nbytes, st_ptr), "shine_octree_sort_new_keys")
        mortons = []
        for l in range(L):
            m = torch.empty(max(c_corners[l], 1), dtype=torch.int64, device=dev)
            plan.lv[l].corner_morton_out = m.data_ptr()
            mortons.append(m)
        if total:
            _abi.check(lib.shine_octree_assign_rows(C.byref(plan), _abi.ptr(sorted_keys), total, st_ptr),
                       "shine_octree_assign_rows")
        new_keys = sorted_keys[total:]                                         # Morton order per level, after fill_nodes
        overflow = torch.zeros(1, dtype=torch.int32, device=dev)
        _abi.check(lib.shine_octree_fill_nodes(C.byref(plan), _abi.ptr(new_keys), n_new, _abi.ptr(overflow), st_ptr),
                   "shine_octree_fill_nodes")
        start = 0
        for l, lvl in enumerate(levels):          # ascending levels: the reference's randn call order (:139,153)
            if c_nodes[l] == 0:
                continue
            st = self._levels[lvl]
            first = st.corner_morton_by_row.numel() == 0 and len(self.hier_features) <= l
            self._grow_features(l, c_corners[l], first, incremental_on, dev)
            st.corner_morton_by_row = torch.cat((st.corner_morton_by_row, mortons[l][:c_corners[l]]))
            st.node_keys = torch.cat((st.node_keys, new_keys[start:start + c_nodes[l]]))
            st.node_ids = torch.cat((st.node_ids, keep[l][1][:c_nodes[l]]))
            st.hash_count = int(st.node_keys.numel())
            st.corner_hash_count = int(st.corner_morton_by_row.numel())
            start += c_nodes[l]
        if int(overflow.item()):
            raise _abi.ShineB200Error("node table overflow while growing the octree")
        self._dict_cache = None
        self._desc_cache = {}
        self._hier_idx = []
        self._last_coord = None

    def _ensure_level_tables(self, st, lvl):
        """Device tables of a level that lost them (unpickled / moved): rebuild from the authoritative arrays."""
        if st.node_keys.numel() and (st.hash is None or st.hash_count != st.node_keys.numel()):
            self._ensure_hash()
        if st.corner_morton_by_row.numel() and (st.corner_hash is None or
                                                st.corner_hash_count != st.corner_morton_by_row.numel()):
            st.corner_hash = None
            self._reserve_corner_table(st, int(st.corner_morton_by_row.numel()))

    def _reserve_node_table(self, st, lvl, n_total):
        """Room for n_total nodes at the usual load factor; growing re-inserts the existing nodes."""
        spn = max(1, int(self._HASH_SLOTS_PER_NODE))
        if st.hash is not None and spn * n_total <= 2 * st.hash_capacity and n_total + 1 <= st.hash_capacity:
            return
        dev = st.node_keys.device
        st.hash_capacity = _next_pow2(max(spn * max(n_total, 1), n_total + 1))
        st.hash = torch.full((st.hash_capacity * _abi.HASH_SLOT_BYTES,), 0xFF, dtype=torch.uint8, device=dev)
        n_old = int(st.node_keys.numel())
        if n_old:
            overflow = torch.zeros(1, dtype=torch.int32, device=dev)
            _abi.check(_abi.lib().shine_hash_insert(_abi.ptr(st.hash), st.hash_capacity, _abi.ptr(st.node_keys.contiguous()),
                                                    _abi.ptr(st.node_ids.contiguous()), n_old, 0, _abi.ptr(overflow),
                                                    _abi.stream_ptr(dev)), "shine_hash_insert")
        st.hash_count = n_old

    def _reserve_corner_table(self, st, n_total):
        if st.corner_hash is not None and 2 * n_total <= st.corner_hash_capacity:
            return
        dev = st.node_keys.device
        st.corner_hash_capacity = _next_pow2(4 * max(n_total, 1))
        st.corner_hash = torch.full((st.corner_hash_capacity * 2,), -1, dtype=torch.int64, device=dev)
        rows = int(st.corner_morton_by_row.numel())
        if rows:
            _abi.check(_abi.lib().shine_octree_corner_rehash(_abi.ptr(st.corner_hash), st.corner_hash_capacity,
                                                             _abi.ptr(st.corner_morton_by_row.contiguous()), rows,
                                                             _abi.stream_ptr(dev)), "shine_octree_corner_rehash")
        st.corner_hash_count = rows

    def interpolat(self, x, level, polynomial_on=True):
        """The 8 blend weights as a tensor (reference :172-196) — kept for API parity; the kernels compute
        the same expression in registers."""
        coords = (2 ** level) * (x * 0.5 + 0.5)
        d = torch.frac(coords)
        t = 3 * (d ** 2) - 2 * (d ** 3) if polynomial_on else d
        tx, ty, tz = t[:, 0], t[:, 1], t[:, 2]
        ux, uy, uz = 1 - tx, 1 - ty, 1 - tz
        p = torch.stack((ux * uy * uz, ux * uy * tz, ux * ty * uz, ux * ty * tz,
                         tx * uy * uz, tx * uy * tz, tx * ty * uz, tx * ty * tz), 0)
        return p.T.unsqueeze(2)

    # ---- device tables -------------------------------------------------------------------------------------

    def _ensure_hash(self):
        """(Re)build / extend the device hash tables so they hold every node (load factor <= 0.5)."""
        lib = _abi.lib()
        for i in range(self.free_level_num, self.max_level + 1):
            st = self._levels[i]
            n = st.node_keys.numel()
            if st.hash is not None and st.hash_count == n:
                continue
            _abi.require_cuda(st.node_keys, "FeatureOctree device tables")
            start = st.hash_count
            spn = max(1, int(self._HASH_SLOTS_PER_NODE))
            # grow when the load factor would pass 2/spn, and always keep at least one empty slot (a full table
            # would turn every miss into a walk over the whole table)
            if st.hash is None or spn * n > 2 * st.hash_capacity or n + 1 > st.hash_capacity:
                st.hash_capacity = _next_pow2(max(spn * max(n, 1), n + 1))
                st.hash = torch.full((st.hash_capacity * _abi.HASH_SLOT_BYTES,), 0xFF, dtype=torch.uint8,
                                     device=st.node_keys.device)
                start = 0
            keys = st.node_keys[start:].contiguous()
            ids = st.node_ids[start:].contiguous()
            overflow = torch.zeros(1, dtype=torch.int32, device=keys.device)
            _abi.check(lib.shine_hash_insert(_abi.ptr(st.hash), st.hash_capacity, _abi.ptr(keys), _abi.ptr(ids),
                                             n - start, start, _abi.ptr(overflow), _abi.stream_ptr(keys.device)),
                       "shine_hash_insert")
            dropped = int(overflow.item())     # once per update(), never inside the training loop
            if dropped:
                raise _abi.ShineB200Error(f"device node table of level {i} overflowed: {dropped} of {n - start} keys "
                                          f"were not stored (capacity {st.hash_capacity})")
            st.hash_count = n
            self._desc_cache = {}

    # open addressing, linear probing: capacity = pow2 >= SLOTS_PER_NODE * nodes at (re)build time, rebuilt when the
    # load factor would exceed 2/SLOTS_PER_NODE.  4 -> load factor <= 0.25..0.5: ~1.2 probes per hit, ~1.4 per miss
    _HASH_SLOTS_PER_NODE = int(os.environ.get("SHINE_HASH_SLOTS_PER_NODE", "4"))

    # Same-address red.add serialises in L2: a level with few rows that receives many updates per step is
    # privatised into R replicas (R = pow2, chosen so that a row sees about _REPLICA_TARGET updates per replica).
    _REPLICA_TARGET = int(os.environ.get("SHINE_REPLICA_TARGET", "512"))
    _REPLICA_MAX = int(os.environ.get("SHINE_REPLICA_MAX", "32"))

    def _replicas_for(self, k: int, rows: int, n_points: int, device) -> tuple[int, torch.Tensor | None]:
        want = (8 * n_points) // max(1, rows * self._REPLICA_TARGET)
        r = 1
        while r * 2 <= min(want, self._REPLICA_MAX):
            r *= 2
        if r <= 1:
            return 1, None
        need = (r - 1) * rows * self.feature_dim
        buf = self._grad_scratch.get(k)
        if buf is None or buf.numel() < need or buf.device != device:
            buf = torch.zeros((self._REPLICA_MAX - 1) * rows * self.feature_dim, dtype=torch.float32, device=device)
            self._grad_scratch[k] = buf
        return r, buf

    def _reduce_replicas(self, desc, device) -> None:
        if any(desc.lv[i].num_replicas > 1 for i in range(desc.num_levels)):
            _abi.check(_abi.lib().shine_reduce_grad_replicas(C.byref(desc), _abi.stream_ptr(device)),
                       "shine_reduce_grad_replicas")

    def _descriptor(self, tables=None, grads=None, n_points: int = 0) -> _abi.ShineOctree:
        """C descriptor, bottom-up like hierarchical_indices (lv[0] = leaf).  With grads and n_points, small hot
        levels get gradient replicas (call _reduce_replicas after the backward kernel)."""
        if self.is_empty():
            raise _abi.ShineB200Error("FeatureOctree is empty: call update() before querying")
        self._ensure_hash()
        tables = list(self.hier_features) if tables is None else list(tables)
        # building the ctypes struct costs ~20 us of Python: reuse it while the same buffers are passed
        # (the signature carries shapes and capacities too: the caching allocator may hand a re-grown table the
        # address of an old one)
        sig = (tuple((t.data_ptr(), t.shape[0]) for t in tables),
               tuple(g.data_ptr() if g is not None else 0 for g in grads) if grads is not None else None, n_points,
               tuple((st.hash.data_ptr(), st.hash_capacity) for st in self._levels if st.hash is not None))
        cache = getattr(self, "_desc_cache", None)
        if not isinstance(cache, dict):
            cache = self._desc_cache = {}
        hit = cache.get(sig)
        if hit is not None:
            return hit
        d = _abi.ShineOctree()
        d.num_levels = self.featured_level_num
        d.feature_dim = self.feature_dim
        d.poly_interp = 1 if self.polynomial_interpolation else 0
        for i in range(self.featured_level_num):
            level = self.max_level - i
            k = self.featured_level_num - i - 1
            st = self._levels[level]
            t = tables[k]
            _abi.require_cuda(t, "FeatureOctree.hier_features")
            if not t.is_contiguous() or t.dtype != torch.float32:
                raise _abi.ShineB200Error("hier_features must be contiguous fp32")
            lv = d.lv[i]
            lv.hash_slots = st.hash.data_ptr()
            lv.features = t.data_ptr()
            lv.feature_grads = grads[k].data_ptr() if grads is not None and grads[k] is not None else None
            lv.hash_capacity = st.hash_capacity
            lv.rows = t.shape[0]
            lv.level = level
            if lv.feature_grads and n_points:
                r, buf = self._replicas_for(k, t.shape[0], n_points, t.device)
                if r > 1:
                    lv.num_replicas, lv.grad_replicas = r, buf.data_ptr()
        if len(cache) >= 8:      # forward / train / indices descriptors alternate inside one loop iteration
            cache.clear()
        cache[sig] = d
        return d

    def _prep_coord(self, coord):
        _abi.require_cuda(coord, "FeatureOctree query")
        if coord.dtype != torch.float32 or not coord.is_contiguous():
            coord = coord.float().contiguous()
        return coord

    def _compute_indices(self, coord):
        coord = self._prep_coord(coord.detach())
        n = coord.shape[0]
        out = torch.empty(self.featured_level_num, n, 8, dtype=torch.int64, device=coord.device)
        desc = self._descriptor()
        _abi.check(_abi.lib().shine_get_indices(C.byref(desc), _abi.ptr(coord), n, _abi.ptr(out),
                                                _abi.stream_ptr(coord.device)), "shine_get_indices")
        return list(out.unbind(0))

    def get_indices(self, coord):
        """Bottom-up list of [N,8] int64 corner rows, -1 x8 where the voxel is not in the tree (reference
        :199-218) — one GPU hash probe per (point, level) instead of N Python dict.get calls."""
        self._hier_idx = self._compute_indices(coord)
        self._last_coord = None
        return self._hier_idx

    def get_indices_fast(self, coord):
        """Reference :267-286 dedupes voxels on the host to save dict lookups; on the GPU every probe is O(1),
        so this is get_indices."""
        return self.get_indices(coord)

    def query_feature_with_indices(self, coord, hierarchical_indices):
        """Blend with caller-supplied indices (reference :222-234).  Plain torch gather on the device — kept for
        API parity (`cal_feature_importance`-style callers); the hot path is `query_feature`."""
        total = torch.zeros(coord.shape[0], self.feature_dim, device=coord.device)
        for i in range(self.featured_level_num):
            level = self.max_level - i
            k = self.featured_level_num - i - 1
            w = self.interpolat(coord, level, self.polynomial_interpolation)
            total = total + (self.hier_features[k][hierarchical_indices[i]] * w).sum(1)
        return total

    def query_feature(self, coord, faster=False):
        """All-in-one feature query (reference :237-244): one kernel that hashes the point into each level,
        gathers the 8 corner rows, blends and sums over levels; autograd scatter-adds into the tables."""
        self.set_zero()
        coord = self._prep_coord(coord)
        self._last_coord = coord
        self._hier_idx = []
        return _QueryFeature.apply(self, coord, *self.hier_features)

    def cal_regularization(self):
        """Continual-learning regulariser (reference :246-255)."""
        regularization = 0.
        idx = self.hierarchical_indices
        for i in range(self.featured_level_num):
            k = self.featured_level_num - i - 1
            unique_indices = idx[i].flatten().unique()
            difference = self.hier_features[k][unique_indices] - self.features_last_frame[k][unique_indices]
            regularization += (self.importance_weight[k][unique_indices] * (difference ** 2)).sum()
        return regularization

    def print_detail(self):
        print("Current Octomap:")
        total = 0
        for level in range(self.featured_level_num):
            size = self.leaf_vox_size * (2 ** (self.featured_level_num - 1 - level))
            count = self.hier_features[level].shape[0]
            print("%.2f m: %d voxel corners" % (size, count))
            total += count
        print("memory: %d x %d x 4 = %.3f MB" % (total, self.feature_dim, total * self.feature_dim * 4 / 1024 / 1024))
        print("--------------------------------")
