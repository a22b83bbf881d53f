// shine_octree_build.cu — FeatureOctree.update (reference model/feature_octree.py:114-166) on the GPU.
//
// The reference grows the map with Python dict loops: per featured level it finds the nodes of the new scan that are
// not in nodes_lookup_tables yet (:123-128), makes their corners unique in lexicographic order (:131-132), numbers the
// unseen corners after the existing rows in that order (:135-151) and stores each new node's 8 corner rows (:162-166).
// The new nodes are inserted in the order kaolin's SPC lists them, which is ascending Morton order (:122,164-166): that
// is the iteration order of nodes_lookup_tables, of get_octree_nodes() and the ordinal of every node.
// Here every step is a kernel over the scan's points / new nodes / new corners, all featured levels at once:
//   1. shine_octree_frame_nodes   per (point, level): key -> frame-local key set; first arrival that is also absent
//                                 from the level's node table appends (node tag | level | key) to ONE list
//   2. shine_octree_frame_corners per (new node, corner): lexicographic corner key -> frame-local set; first arrival
//                                 absent from the level's corner table appends (level | key) to ONE list, placed by
//                                 the host right after a copy of the node list
//   3. shine_octree_sort_new_keys radix sort of both lists at once (CUB): corners first (node tag clear), level-major,
//                                 lexicographic inside a level = the reference's row order; then the nodes, level-major,
//                                 Morton order inside a level = the reference's insertion order.  One sort instead of
//                                 two keeps the per-frame launch count down (a onesweep sort is ~16 launches).
//   4. shine_octree_assign_rows   row = rows_before[level] + rank inside the level; insert into the corner table
//   5. shine_octree_fill_nodes    8 corner rows of every new node -> node table slot, ordinal = nodes_before[level] +
//                                 rank inside the level, + the flat arrays behind the dict views
// The host reads two small count vectors in between (it must size the new feature rows anyway).
#include <cub/device/device_radix_sort.cuh>

#include "shine_device.cuh"

namespace {

struct CornerSlot { unsigned long long key; int32_t row; int32_t pad; };
static_assert(sizeof(CornerSlot) == 16, "corner slot is 16 bytes");

// World levels up to 15: kaolin quantises to int16 (the reference cannot go further either), and spread3 / the stored
// Morton codes keep 16 bits per axis, which holds the corner coordinates 0 .. 2^15 of level 15.
constexpr int kMaxWorldLevel = 15;
constexpr int kLexBits = 16;                                   // corner coordinate bits per axis in the lexicographic key
constexpr unsigned long long kLexMask = (1ull << (3 * kLexBits)) - 1ull;
constexpr int kNodeKeyBits = 3 * kMaxWorldLevel;               // node Morton keys: 45 bits
constexpr unsigned long long kNodeKeyMask = (1ull << kNodeKeyBits) - 1ull;
constexpr int kLevelTagBits = 3;                               // level index 0 .. SHINE_MAX_LEVELS - 1
constexpr int kNodeTagBit = 3 * kLexBits + kLevelTagBits;      // set on node entries of the sort: they sort after corners
constexpr int kSortBits = kNodeTagBit + 1;
static_assert(kNodeKeyBits + kLevelTagBits <= kNodeTagBit, "node entries fit below the node tag");
static_assert(SHINE_MAX_LEVELS <= (1 << kLevelTagBits), "level index fits its tag");

__host__ __device__ __forceinline__ unsigned long long node_entry(int l, unsigned long long key) {
    return (1ull << kNodeTagBit) | ((unsigned long long)l << kNodeKeyBits) | key;
}
__host__ __device__ __forceinline__ int node_entry_level(unsigned long long e) {
    return (int)((e >> kNodeKeyBits) & ((1u << kLevelTagBits) - 1u));
}

// index of the first sorted entry of level l (entries of levels < l come first): j - level_start = rank inside the level
__device__ __forceinline__ int level_start(const int32_t* counts, int l) {
    int start = 0;
    for (int q = 0; q < l; ++q) start += counts[q];
    return start;
}

// Lexicographic key of a corner, ordered as torch.unique(dim=0) orders kaolin's int16 corner points (:131-132): a corner
// coordinate of 2^15 (the + face at world level 15) wraps to -2^15 there and comes first.  c ^ 0x8000 maps the int16
// order onto unsigned 16-bit order; below level 15 it keeps the plain order.
__host__ __device__ __forceinline__ unsigned long long lex_key(uint32_t x, uint32_t y, uint32_t z) {
    return ((unsigned long long)(x ^ 0x8000u) << (2 * kLexBits)) | ((unsigned long long)(y ^ 0x8000u) << kLexBits) |
           (unsigned long long)(z ^ 0x8000u);
}
// coordinate `axis` (0 = x) of a lexicographic key
__host__ __device__ __forceinline__ uint32_t lex_coord(unsigned long long lk, int axis) {
    return ((uint32_t)(lk >> ((2 - axis) * kLexBits)) & 0xFFFFu) ^ 0x8000u;
}

__device__ __forceinline__ uint32_t compact3(unsigned long long v) {       // inverse of spread3
    v &= 0x249249249249ull;
    v = (v | (v >> 2)) & 0x0C30C30C30C3ull;
    v = (v | (v >> 4)) & 0x00F00F00F00Full;
    v = (v | (v >> 8)) & 0x0000FF0000FFull;
    v = (v | (v >> 16)) & 0xFFFFull;
    return (uint32_t)v;
}

// insert into a key-only set; true when this call created the entry
__device__ __forceinline__ bool set_insert(unsigned long long* set, uint32_t mask, unsigned long long key) {
    uint32_t h = hash_key(key) & mask;
    for (uint32_t it = 0; it <= mask; ++it) {
        const unsigned long long prev = atomicCAS(&set[h], kEmptyKey, key);
        if (prev == kEmptyKey) return true;
        if (prev == key) return false;
        h = (h + 1) & mask;
    }
    return false;    // full (the host sizes the sets at twice the number of insertions: cannot happen)
}

__device__ __forceinline__ int corner_lookup(const CornerSlot* tab, uint32_t mask, unsigned long long key) {
    uint32_t h = hash_key(key) & mask;
    for (uint32_t it = 0; it <= mask; ++it) {
        const unsigned long long k = tab[h].key;
        if (k == key) return tab[h].row;
        if (k == kEmptyKey) return -1;
        h = (h + 1) & mask;
    }
    return -1;
}

__global__ void __launch_bounds__(256) frame_nodes_kernel(const __grid_constant__ shine_build plan,
                                                          const float* __restrict__ pts, int64_t n) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const unsigned long long leaf = morton_of(pts[3 * i], pts[3 * i + 1], pts[3 * i + 2], plan.max_level);
    for (int l = 0; l < plan.num_levels; ++l) {
        const shine_build_level& b = plan.lv[l];
        const unsigned long long key = leaf >> (3 * (plan.max_level - b.level));      // ancestors by shift (:116-122)
        if (!set_insert(reinterpret_cast<unsigned long long*>(b.frame_node_set), b.frame_node_set_capacity - 1, key)) continue;
        if (b.node_slots && b.nodes_before > 0 &&
            probe_slot(reinterpret_cast<const HashSlot*>(b.node_slots), b.node_capacity - 1, key) >= 0)
            continue;                                                                   // seen in an earlier frame (:124-127)
        const int pos = atomicAdd(plan.new_node_total, 1);
        atomicAdd(plan.new_node_count + l, 1);
        plan.new_node_keys[pos] = node_entry(l, key);                                 // arrival order; sorted in step 3
    }
}

__global__ void __launch_bounds__(256) frame_corners_kernel(const __grid_constant__ shine_build plan, int total_nodes) {
    for (int64_t gt = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; gt < (int64_t)total_nodes * 8;
         gt += (int64_t)gridDim.x * blockDim.x) {
        const unsigned long long e = plan.new_node_keys[gt >> 3];
        const int l = node_entry_level(e);
        const shine_build_level& b = plan.lv[l];
        const unsigned long long key = e & kNodeKeyMask;
        const int c = (int)(gt & 7);
        const uint32_t x = compact3(key >> 2) + ((c >> 2) & 1), y = compact3(key >> 1) + ((c >> 1) & 1), z = compact3(key) + (c & 1);
        const unsigned long long lk = lex_key(x, y, z);                                 // points_to_corners order (:131)
        if (!set_insert(reinterpret_cast<unsigned long long*>(b.frame_corner_set), b.frame_corner_set_capacity - 1, lk)) continue;
        if (b.corner_slots && b.rows_before > 0 &&
            corner_lookup(reinterpret_cast<const CornerSlot*>(b.corner_slots), b.corner_capacity - 1, lk) >= 0)
            continue;                                                                   // existing corner keeps its row (:148)
        const int pos = atomicAdd(plan.new_corner_total, 1);
        atomicAdd(plan.new_corner_count + l, 1);
        plan.new_corner_keys[pos] = ((unsigned long long)l << (3 * kLexBits)) | lk;
    }
}

__global__ void __launch_bounds__(256) assign_rows_kernel(const __grid_constant__ shine_build plan,
                                                          const unsigned long long* __restrict__ sorted, int total) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= total) return;
    const unsigned long long tagged = sorted[j];
    const int l = (int)(tagged >> (3 * kLexBits));
    const unsigned long long lk = tagged & kLexMask;
    const int start = level_start(plan.new_corner_count, l);
    const shine_build_level& b = plan.lv[l];
    const int row = b.rows_before + (j - start);                                       // append-only, lexicographic (:135-151)
    CornerSlot* tab = reinterpret_cast<CornerSlot*>(b.corner_slots);
    const uint32_t mask = b.corner_capacity - 1;
    uint32_t h = hash_key(lk) & mask;
    for (uint32_t it = 0; it <= mask; ++it) {
        const unsigned long long prev = atomicCAS(&tab[h].key, kEmptyKey, lk);
        if (prev == kEmptyKey) { tab[h].row = row; break; }
        h = (h + 1) & mask;
    }
    b.corner_morton_out[j - start] =
        (int64_t)((spread3(lex_coord(lk, 0)) << 2) | (spread3(lex_coord(lk, 1)) << 1) | spread3(lex_coord(lk, 2)));
}

// sorted: the node part of the sort output (level-major, Morton order inside a level).  The tag is stripped in place, so
// the host can append each level's slice to node_keys as it is.
__global__ void __launch_bounds__(256) fill_nodes_kernel(const __grid_constant__ shine_build plan, unsigned long long* __restrict__ sorted,
                                                         int total_nodes, int32_t* overflow) {
    for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < total_nodes; j += gridDim.x * blockDim.x) {
        const unsigned long long e = sorted[j];
        const int l = node_entry_level(e);
        const shine_build_level& b = plan.lv[l];
        const int k = j - level_start(plan.new_node_count, l);                          // reference insertion order (:164-166)
        const unsigned long long key = e & kNodeKeyMask;
        const uint32_t x0 = compact3(key >> 2), y0 = compact3(key >> 1), z0 = compact3(key);
        int ids[8];
#pragma unroll
        for (int c = 0; c < 8; ++c)
            ids[c] = corner_lookup(reinterpret_cast<const CornerSlot*>(b.corner_slots), b.corner_capacity - 1,
                                   lex_key(x0 + ((c >> 2) & 1), y0 + ((c >> 1) & 1), z0 + (c & 1)));
        HashSlot* slots = reinterpret_cast<HashSlot*>(b.node_slots);
        const uint32_t mask = b.node_capacity - 1, h0 = hash_key(key) & mask;
        bool stored = false;
        for (uint32_t it = 0; it <= mask && !stored; ++it) {
            const uint32_t h = probe_pos(h0, it, mask);
            const unsigned long long prev = atomicCAS(&slots[h].key, kEmptyKey, key);
            if (prev == kEmptyKey || prev == key) {
                slots[h].node = b.nodes_before + k;
                slots[h].key2 = key;
#pragma unroll
                for (int c = 0; c < 4; ++c) { slots[h].ids0[c] = ids[2 * c]; slots[h].ids1[c] = ids[2 * c + 1]; }
                note_displacement(slots, h0, it);
                stored = true;
            }
        }
        if (!stored && overflow) atomicAdd(overflow, 1);
        sorted[j] = key;
#pragma unroll
        for (int c = 0; c < 8; ++c) b.node_ids_out[(int64_t)k * 8 + c] = ids[c];
    }
}

// re-insert rows [0, n) of a level into a fresh corner table: key from the row's Morton code
__global__ void __launch_bounds__(256) corner_rehash_kernel(CornerSlot* tab, uint32_t mask, const int64_t* __restrict__ morton_by_row,
                                                            int64_t n) {
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n) return;
    const unsigned long long m = (unsigned long long)morton_by_row[r];
    const unsigned long long lk = lex_key(compact3(m >> 2), compact3(m >> 1), compact3(m));
    uint32_t h = hash_key(lk) & mask;
    for (uint32_t it = 0; it <= mask; ++it) {
        const unsigned long long prev = atomicCAS(&tab[h].key, kEmptyKey, lk);
        if (prev == kEmptyKey) { tab[h].row = (int32_t)r; return; }
        h = (h + 1) & mask;
    }
}

int check_build(const shine_build* p) {
    if (!p || p->num_levels < 1 || p->num_levels > SHINE_MAX_LEVELS || p->max_level < 1 || p->max_level > kMaxWorldLevel)
        return SHINE_ERR_INVALID_ARG;
    if (!p->new_node_count || !p->new_corner_count || !p->new_corner_total || !p->new_node_total || !p->new_node_keys)
        return SHINE_ERR_INVALID_ARG;
    for (int l = 0; l < p->num_levels; ++l) {
        const shine_build_level& b = p->lv[l];
        if (b.level < 1 || b.level > p->max_level) return SHINE_ERR_INVALID_ARG;
        if (!b.frame_node_set || !is_pow2(b.frame_node_set_capacity)) return SHINE_ERR_INVALID_ARG;
    }
    return SHINE_OK;
}

}  // namespace

extern "C" {

int shine_octree_frame_nodes(const shine_build* plan, const float* points, int64_t n, void* stream) {
    int rc = check_build(plan);
    if (rc) return rc;
    if (n < 0 || (n > 0 && !points)) return SHINE_ERR_INVALID_ARG;
    if (n == 0) return SHINE_OK;
    DeviceGuard guard(plan->new_node_count);
    frame_nodes_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(*plan, points, n);
    return (int)cudaGetLastError();
}

int shine_octree_frame_corners(const shine_build* plan, int32_t new_nodes, void* stream) {
    int rc = check_build(plan);
    if (rc) return rc;
    if (new_nodes <= 0) return SHINE_OK;
    for (int l = 0; l < plan->num_levels; ++l)
        if (!plan->lv[l].frame_corner_set || !is_pow2(plan->lv[l].frame_corner_set_capacity)) return SHINE_ERR_INVALID_ARG;
    if (!plan->new_corner_keys) return SHINE_ERR_INVALID_ARG;
    DeviceGuard guard(plan->new_node_count);
    int64_t blocks = ((int64_t)new_nodes * 8 + 255) / 256;
    const int64_t cap = (int64_t)sm_count() * 8;
    if (blocks > cap) blocks = cap;
    frame_corners_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(*plan, new_nodes);
    return (int)cudaGetLastError();
}

int64_t shine_octree_sort_scratch_bytes(int32_t n) {
    size_t bytes = 0;
    cub::DeviceRadixSort::SortKeys(nullptr, bytes, (const unsigned long long*)nullptr, (unsigned long long*)nullptr,
                                   n > 0 ? n : 1, 0, kSortBits);
    return (int64_t)bytes;
}

int shine_octree_sort_new_keys(const void* keys_in, void* keys_out, int32_t n, void* scratch, int64_t scratch_bytes, void* stream) {
    if (n < 0 || (n > 0 && (!keys_in || !keys_out || !scratch))) return SHINE_ERR_INVALID_ARG;
    if (n == 0) return SHINE_OK;
    DeviceGuard guard(keys_out);
    size_t bytes = (size_t)scratch_bytes;
    return (int)cub::DeviceRadixSort::SortKeys(scratch, bytes, (const unsigned long long*)keys_in, (unsigned long long*)keys_out, n,
                                               0, kSortBits, (cudaStream_t)stream);
}

int shine_octree_assign_rows(const shine_build* plan, const void* sorted_keys, int32_t total, void* stream) {
    int rc = check_build(plan);
    if (rc) return rc;
    if (total < 0 || (total > 0 && !sorted_keys)) return SHINE_ERR_INVALID_ARG;
    if (total == 0) return SHINE_OK;
    for (int l = 0; l < plan->num_levels; ++l) {
        const shine_build_level& b = plan->lv[l];
        if (!b.corner_slots || !is_pow2(b.corner_capacity) || !b.corner_morton_out) return SHINE_ERR_INVALID_ARG;
    }
    DeviceGuard guard(plan->new_node_count);
    assign_rows_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
        *plan, (const unsigned long long*)sorted_keys, total);
    return (int)cudaGetLastError();
}

int shine_octree_fill_nodes(const shine_build* plan, void* sorted_nodes, int32_t new_nodes, int32_t* overflow_count,
                            void* stream) {
    int rc = check_build(plan);
    if (rc) return rc;
    if (new_nodes < 0 || (new_nodes > 0 && !sorted_nodes)) return SHINE_ERR_INVALID_ARG;
    if (new_nodes == 0) return SHINE_OK;
    for (int l = 0; l < plan->num_levels; ++l) {
        const shine_build_level& b = plan->lv[l];
        if (!b.node_slots || !is_pow2(b.node_capacity) || !b.corner_slots || !is_pow2(b.corner_capacity) || !b.node_ids_out)
            return SHINE_ERR_INVALID_ARG;
    }
    DeviceGuard guard(plan->new_node_count);
    int64_t blocks = ((int64_t)new_nodes + 255) / 256;
    const int64_t cap = (int64_t)sm_count() * 8;
    if (blocks > cap) blocks = cap;
    fill_nodes_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(*plan, (unsigned long long*)sorted_nodes, new_nodes,
                                                                        overflow_count);
    return (int)cudaGetLastError();
}

int shine_octree_corner_rehash(void* corner_slots, uint32_t capacity, const int64_t* corner_morton_by_row, int64_t rows, void* stream) {
    if (!corner_slots || !is_pow2(capacity) || rows < 0 || (rows > 0 && !corner_morton_by_row)) return SHINE_ERR_INVALID_ARG;
    if (rows == 0) return SHINE_OK;
    DeviceGuard guard(corner_slots);
    corner_rehash_kernel<<<(unsigned)((rows + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
        reinterpret_cast<CornerSlot*>(corner_slots), capacity - 1, corner_morton_by_row, rows);
    return (int)cudaGetLastError();
}

}  // extern "C"
