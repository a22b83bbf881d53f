"""Host restatements of the spatial partition's exchange (partition.BoundaryPlan, csrc/shine_comm.cu, csrc/shine_p2p.cu)
and the per-element error bound of a partitioned training step.  Test infrastructure, no GPU needed.

Plan.  For per-rank, per-level corner key sets, `check_plans` states what every rank's BoundaryPlan must hold: a level's
shared corners are the keys listed by two or more ranks, in ascending key order (the agreed slot order); `slots` are
unique with `inverse[slots] == rows` and -1 elsewhere; `holders` has bit r set exactly for the ranks that list the key;
`owned` marks the rows whose rank is the corner's lowest holder; the levels' segments follow the decoder segment back to
back; and every rank agrees on counts, offsets and holders.

Exchange.  Both routes leave the same values in the decoder segment and in every shared corner's rows: the fp32 sum,
from +0.0, over the corner's holders in rank order 0, 1, ... (the decoder segment: over every rank).  The NCCL route packs
every rank's rows at their slots into a zeroed buffer and sums all ranks; the peer-memory kernel reads only the holders.
Adding +0 is exact and the running sum starts at +0 (never -0), so the two agree bit for bit: `exchange_model`.

Bound of a partitioned step.  Rank r trains its share of ONE global batch, every per-point gradient scaled by 1/n_global,
and the exchange sums the ranks' partials of every shared row.  Against the fp64 step of the global batch
(tests/test_gpu_replicas.Ref), row u, channel f:
    |got - want64| <= (sum_r k_u^(r) + h_u - 1 + C) u S_u + T_u
S_u and T_u are sums over the points that touch u, so they do not depend on the split and come from the global Ref.
k_u^(r) counts the fp32 adds rank r's step makes into its partial of u: the (point, corner) terms of its points for the
per-point kernels (a replica fold only regroups those terms: test_gpu_replicas' docstring), `error_bound.grouped_counts`
over the rank's own tiles for the Morton-ordered grouped kernel, plus R - 1 where that kernel's fold ran.  h_u is the
number of ranks that hold a row of u: the exchange adds h_u partials into +0, h_u - 1 roundings.  The decoder gradients
take the model of tests/decoder_bound.py at depth max_r kernel_depth(n_r) + world - 1 (each rank's kernel, then the
world - 1 adds of the exchange), and the loss `infer_bound.LossRef` with world - 1 more adds per term.
"""
from __future__ import annotations

import numpy as np
import torch

from tests.error_bound import C_SLACK, U, grade_tables, grouped_counts


# ---- the plan ------------------------------------------------------------------------------------------------------------

def shared_keys(per_rank_level_keys, lvl):
    """(sorted shared keys, holder mask per shared key) of one level, by plain set arithmetic."""
    holders: dict[int, int] = {}
    for r, levels in enumerate(per_rank_level_keys):
        for k in np.asarray(levels[lvl].cpu()).tolist():
            holders[k] = holders.get(k, 0) | (1 << r)
    keys = sorted(k for k, m in holders.items() if bin(m).count("1") >= 2)
    return np.array(keys, dtype=np.int64), np.array([holders[k] for k in keys], dtype=np.int64)


def check_plans(plans, per_rank_level_keys, feature_dim, dec_floats):
    """Every invariant of the module docstring for the plans of every rank (plans[r] built for rank r)."""
    world = len(per_rank_level_keys)
    n_levels = len(per_rank_level_keys[0])
    for r, p in enumerate(plans):
        assert p.rank == r and p.world == world and p.feature_dim == feature_dim and p.dec_floats == dec_floats
        off = dec_floats
        for lvl in range(n_levels):
            shared, held = shared_keys(per_rank_level_keys, lvl)
            mine = np.asarray(per_rank_level_keys[r][lvl].cpu())
            rows, slots = p.rows[lvl].cpu().numpy(), p.slots[lvl].cpu().numpy()
            inv, owned = p.inverse[lvl].cpu().numpy(), p.owned[lvl].cpu().numpy()
            hol = p.holders[lvl].cpu().numpy()
            what = f"rank {r} level {lvl}"
            assert p.counts[lvl] == shared.size, f"{what}: {p.counts[lvl]} slots, {shared.size} shared keys"
            assert p.offsets[lvl] == off, f"{what}: offset {p.offsets[lvl]}, expected {off}"
            off += shared.size * feature_dim
            assert hol.dtype == np.int32 and np.array_equal(hol.astype(np.int64) & 0xFFFFFFFF, held), f"{what}: holders"
            assert all(bin(int(m)).count("1") >= 2 for m in held)
            # rows: exactly the local rows whose key is shared, each at the slot of its key
            want_rows = np.flatnonzero(np.isin(mine, shared))
            assert np.array_equal(np.sort(rows), want_rows), f"{what}: rows are not the shared local rows"
            assert np.unique(slots).size == slots.size, f"{what}: a slot is listed twice"
            assert np.array_equal(shared[slots], mine[rows]), f"{what}: a row sits at another key's slot"
            want_inv = np.full(shared.size, -1, dtype=np.int64)
            want_inv[slots] = rows
            assert inv.shape == (shared.size,) and np.array_equal(inv, want_inv), f"{what}: inverse"
            assert all((int(held[s]) >> r) & 1 for s in slots), f"{what}: a row of a corner whose holders omit the rank"
            lowest = np.array([(int(m) & -int(m)).bit_length() - 1 for m in held[slots]], dtype=np.int64)
            assert np.array_equal(owned, lowest == r), f"{what}: owned is not 'lowest holder'"
        assert p.total_floats == off, f"rank {r}: total_floats {p.total_floats}, expected {off}"
    for p in plans[1:]:
        assert p.counts == plans[0].counts and p.offsets == plans[0].offsets
        assert p.total_floats == plans[0].total_floats
        assert all(torch.equal(a.cpu(), b.cpu()) for a, b in zip(p.holders, plans[0].holders))


def holders_per_float(plan):
    """[total_floats] int64 holder mask of every float of the exchange buffer (decoder segment: every rank)."""
    m = np.full(plan.total_floats, (1 << plan.world) - 1, dtype=np.int64)
    for lvl, n in enumerate(plan.counts):
        seg = slice(plan.offsets[lvl], plan.offsets[lvl] + n * plan.feature_dim)
        m[seg] = np.repeat(plan.holders[lvl].cpu().numpy().astype(np.int64), plan.feature_dim)
    return m


def exchange_model(bufs, plan):
    """The exchange's result for every float of the buffer: fp32 sum from +0 over the holders in rank order.
    bufs: per rank, the [total_floats] fp32 buffer that rank packed (slots of corners it does not hold: anything)."""
    mask = holders_per_float(plan)
    acc = np.zeros(plan.total_floats, dtype=np.float32)
    for r, b in enumerate(bufs):
        b = np.asarray(b, dtype=np.float32)
        acc = acc + np.where((mask >> r) & 1 == 1, b, np.float32(0))
    return acc


def pack_host(plan, tables, total=None):
    """The buffer a rank packs: zeros, its decoder segment left 0, its rows at their slots."""
    buf = np.zeros(plan.total_floats if total is None else total, dtype=np.float32)
    F = plan.feature_dim
    for lvl, t in enumerate(tables):
        seg = buf[plan.offsets[lvl]:plan.offsets[lvl] + plan.counts[lvl] * F].reshape(-1, F)
        seg[plan.slots[lvl].cpu().numpy()] = np.asarray(t)[plan.rows[lvl].cpu().numpy()]
    return buf


# ---- the bound of a partitioned step -------------------------------------------------------------------------------------

def global_rows(keys, key_to_row):
    return np.array([key_to_row[int(k)] for k in np.asarray(keys.cpu() if torch.is_tensor(keys) else keys).tolist()],
                    dtype=np.int64)


class PartitionBound:
    """The bound of the module docstring on top of a global `Ref` (already `for_kernel`-ed for the kernel that ran).
    rank_points[r]: indices into the global batch, in the order rank r's kernel saw them; rank_rows[r][kk]: global row of
    every local row of rank r's table kk (trash row excluded); replicas[r]: R per table (coarse -> fine) of rank r's grouped
    fold, or None."""

    def __init__(self, ref, rank_points, rank_rows, grouped, replicas=None):
        self.ref, self.world = ref, len(rank_points)
        L = len(ref.want)
        self.k, self.h = [], []
        for kk in range(L):
            rows = ref.want[kk].shape[0]
            k = np.zeros(rows, dtype=np.int64)
            for r, idx in enumerate(rank_points):
                ix = ref._ix[kk][np.asarray(idx)]
                if grouped:
                    kr = grouped_counts(ix, rows)
                    R = 1 if replicas is None or replicas[r] is None else replicas[r][kk]
                    kr = kr + np.where(kr > 0, R - 1, 0)
                else:
                    kr = np.bincount(ix[ix >= 0], minlength=rows)
                k += kr
            h = np.zeros(rows, dtype=np.int64)
            for rr in rank_rows:
                h[rr[kk]] += 1
            self.k.append(k + np.maximum(h - 1, 0))
            self.h.append(h)
        self.rank_rows = rank_rows

    def bound(self, kk):
        return (self.k[kk][:, None] + self.ref.slack) * U * self.ref.S[kk] + self.ref.T[kk]

    def grade_rank(self, r, got_tables, what):
        """Every element of rank r's tables (trash row excluded) against the bound of its global row."""
        want, bounds, ks, Ss = [], [], [], []
        for kk, got in enumerate(got_tables):
            rows = self.rank_rows[r][kk]
            assert rows.shape[0] == np.asarray(got).shape[0] - 1, f"{what}: table {kk} has another row count"
            pad = lambda a: np.concatenate((a[rows], np.zeros_like(a[:1])))        # noqa: E731 (trash row: not graded)
            want.append(pad(self.ref.want[kk])); bounds.append(pad(self.bound(kk)))
            ks.append(pad(self.k[kk])); Ss.append(pad(self.ref.S[kk]))
        return grade_tables(got_tables, want, bounds, ks, Ss, what, "partition bounds")

    def decoder_depth(self, sizes, sms=None):
        from tests.decoder_bound import kernel_depth
        return max(kernel_depth(n, 1, sms) if sms else kernel_depth(n) for n in sizes) + self.world - 1

    def loss_ref(self, case):
        from tests.infer_bound import LossRef
        c = case["cfg"]
        return LossRef(self.ref.pred, self.ref.P, case["label"], case["weight"], "sdf_bce", slack=C_SLACK + self.world - 1,
                       sigma=c["sigma"], weighted=c["weighted"], reduction=c["reduction"])
