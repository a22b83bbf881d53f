// shine_pool.cu — the sample pool of incremental mapping with replay (continual.window_replay_on), one launch per frame.
// Reference: dataset/lidar_dataset.py:235-271 (selected at shine_incre.py:106): drop the pool samples that lie
// window_radius_m or more from the new sensor origin (`(coord_pool - origin).norm(2, dim=-1) < r`, three masked gathers),
// then `torch.cat` the frame behind the survivors.  Here both are one in-place stream compaction over the virtual sequence
// [pool's `size` old samples (kept iff inside the window) | frame's `n_new` samples (always kept)], in the reference's order.
//
// Single pass with decoupled look-back: a tile takes its id from an atomic counter (so every tile it looks back at has
// started and the look-back makes progress), reads everything it may have to move, publishes its kept count, then sums
// its predecessors' counts.  Output positions never exceed input positions, and a tile writes only after every earlier
// tile has published, i.e. after they have read their inputs; later tiles read above everything this tile writes.  So the
// compaction can run in place.
#include "shine_device.cuh"

namespace {

constexpr int kPoolThreads = 256;
constexpr int kPoolItems = 8;                          // samples per thread, striped: item k of thread t is k*256 + t
constexpr int kPoolTile = kPoolThreads * kPoolItems;   // 2048 samples per tile
constexpr int kPoolWarps = kPoolThreads / 32;
constexpr int64_t kPoolScratchHeader = 16;             // tile counter, padded; then one status word per tile

// tile status word: flag in the top two bits, number of kept samples in the low 62
constexpr unsigned long long kStatusAggregate = 1ull << 62;   // this tile's own count
constexpr unsigned long long kStatusPrefix = 2ull << 62;      // count of this tile and every tile before it
constexpr unsigned long long kStatusValue = (1ull << 62) - 1;

__device__ __forceinline__ unsigned long long ld_acquire_u64(const unsigned long long* p) {
    unsigned long long v;
    asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}

__device__ __forceinline__ void st_release_u64(unsigned long long* p, unsigned long long v) {
    asm volatile("st.release.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}

struct PoolArgs {
    float* coord;                 // pool [capacity, 3]
    float* label;                 // pool [capacity]
    float* weight;                // pool [capacity]
    const float* new_coord;       // frame [n_new, 3]
    const float* new_label;
    const float* new_weight;
    int64_t size, n_new;
    float ox, oy, oz, r;
    unsigned int* tile_counter;
    unsigned long long* status;   // [tiles], zero (no status yet) on entry
    int64_t* size_out;
};

// The reference's predicate `(coord - origin).norm(2, dim=-1) < r` in fp32 without contraction: (dx^2 + dy^2) + dz^2,
// correctly rounded sqrt, strict <.  A NaN coordinate fails the comparison and is dropped, as in the reference.
__device__ __forceinline__ bool inside_window(float x, float y, float z, const PoolArgs& a) {
    const float dx = __fsub_rn(x, a.ox), dy = __fsub_rn(y, a.oy), dz = __fsub_rn(z, a.oz);
    const float d2 = __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
    return __fsqrt_rn(d2) < a.r;
}

__global__ void __launch_bounds__(kPoolThreads) pool_window_append_kernel(const __grid_constant__ PoolArgs a) {
    __shared__ unsigned int s_tile;
    __shared__ int s_offset[kPoolItems * kPoolWarps];   // kept samples per (item round, warp), then their exclusive scan
    __shared__ int s_count;                             // kept samples of the tile
    __shared__ int s_fast;                              // the exclusive prefix is known before this tile publishes
    __shared__ long long s_prefix;                      // kept samples of all earlier tiles
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) s_tile = atomicAdd(a.tile_counter, 1u);
    __syncthreads();
    const unsigned int tile = s_tile;
    const int64_t begin = (int64_t)tile * kPoolTile;
    const int64_t total = a.size + a.n_new;

    // 1. predicate: old samples read their coordinates; frame samples are always kept
    float x[kPoolItems], y[kPoolItems], z[kPoolItems], lb[kPoolItems], wt[kPoolItems];
    unsigned int ballot[kPoolItems];
    unsigned int kept = 0;
#pragma unroll
    for (int k = 0; k < kPoolItems; ++k) {
        const int64_t i = begin + k * kPoolThreads + tid;
        bool keep = false;
        if (i < a.size) {
            x[k] = a.coord[3 * i]; y[k] = a.coord[3 * i + 1]; z[k] = a.coord[3 * i + 2];
            keep = inside_window(x[k], y[k], z[k], a);
        } else {
            keep = i < total;
        }
        kept |= (unsigned)keep << k;
        ballot[k] = __ballot_sync(kFull, keep);
        if (lane == 0) s_offset[k * kPoolWarps + warp] = __popc(ballot[k]);
    }
    __syncthreads();

    // 2. tile-local exclusive scan of the (round, warp) counts, which is the samples' order; peek at the predecessor
    if (warp == 0) {
        const int c0 = s_offset[2 * lane], c1 = s_offset[2 * lane + 1];
        int incl = c0 + c1;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int v = __shfl_up_sync(kFull, incl, o);
            if (lane >= o) incl += v;
        }
        const int excl = incl - c0 - c1;
        s_offset[2 * lane] = excl;
        s_offset[2 * lane + 1] = excl + c0;
        if (lane == 31) s_count = incl;
        if (lane == 0) {
            // nothing dropped ahead of this tile yet and the predecessor is done: the prefix is `begin`, and the
            // samples that stay where they are need not be read beyond their coordinates
            const unsigned long long prev = tile ? ld_acquire_u64(a.status + tile - 1) : (kStatusPrefix | 0ull);
            const bool fast = (prev & ~kStatusValue) == kStatusPrefix && (int64_t)(prev & kStatusValue) == begin;
            s_fast = fast;
            s_prefix = fast ? begin : -1;
        }
    }
    __syncthreads();
    const bool fast = s_fast;
    const unsigned lt_mask = (1u << lane) - 1u;

    // 3. read what may move.  Without a known prefix every kept sample may move; with it, only those behind a drop.
#pragma unroll
    for (int k = 0; k < kPoolItems; ++k) {
        if (!((kept >> k) & 1u)) continue;
        const int64_t i = begin + k * kPoolThreads + tid;
        if (i >= a.size) {
            const int64_t j = i - a.size;
            x[k] = a.new_coord[3 * j]; y[k] = a.new_coord[3 * j + 1]; z[k] = a.new_coord[3 * j + 2];
            lb[k] = a.new_label[j]; wt[k] = a.new_weight[j];
        } else if (!fast || begin + s_offset[k * kPoolWarps + warp] + __popc(ballot[k] & lt_mask) != i) {
            lb[k] = a.label[i]; wt[k] = a.weight[i];
        }
    }
    // every read of this tile is performed before the status below can let a later tile write over it
    __syncthreads();

    // 4. publish, look back
    if (fast) {
        if (tid == 0) {
            __threadfence();
            st_release_u64(a.status + tile, kStatusPrefix | (unsigned long long)(begin + s_count));
        }
    } else if (warp == 0) {
        if (lane == 0) {
            __threadfence();
            st_release_u64(a.status + tile, kStatusAggregate | (unsigned long long)s_count);
        }
        // a window of 32 predecessors per round, nearest in lane 0; stop at the nearest inclusive prefix
        long long prefix = 0;
        for (int64_t base = (int64_t)tile - 1;; base -= 32) {
            const int64_t t = base - lane;
            unsigned long long s = kStatusPrefix;       // "before tile 0": prefix 0
            if (t >= 0) {
                int spin = 0;
                while (((s = ld_acquire_u64(a.status + t)) & ~kStatusValue) == 0ull) {
                    __nanosleep(32);
                    if (++spin > (1 << 24)) __trap();    // never hang the GPU on a protocol bug
                }
            }
            const unsigned is_prefix = __ballot_sync(kFull, (s & ~kStatusValue) == kStatusPrefix);
            const int stop = is_prefix ? __ffs(is_prefix) - 1 : 31;
            long long v = lane <= stop ? (long long)(s & kStatusValue) : 0ll;
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(kFull, v, o);
            prefix += v;
            if (is_prefix) break;
        }
        if (lane == 0) {
            st_release_u64(a.status + tile, kStatusPrefix | (unsigned long long)(prefix + s_count));
            s_prefix = prefix;
        }
    }
    __syncthreads();
    const int64_t prefix = s_prefix;
    if (tid == 0 && tile == gridDim.x - 1) *a.size_out = prefix + s_count;

    // 5. write the kept samples at their output positions; an old sample whose position does not change is not written
#pragma unroll
    for (int k = 0; k < kPoolItems; ++k) {
        if (!((kept >> k) & 1u)) continue;
        const int64_t i = begin + k * kPoolThreads + tid;
        const int64_t out = prefix + s_offset[k * kPoolWarps + warp] + __popc(ballot[k] & lt_mask);
        if (out == i && i < a.size) continue;
        a.coord[3 * out] = x[k]; a.coord[3 * out + 1] = y[k]; a.coord[3 * out + 2] = z[k];
        a.label[out] = lb[k];
        a.weight[out] = wt[k];
    }
}

int64_t pool_tiles(int64_t n_total) { return (n_total + kPoolTile - 1) / kPoolTile; }

// device memory of `dev`, or (allow_pinned) page-locked host memory the kernel can read through the unified address space
bool pointer_usable(const void* p, int dev, bool allow_pinned) {
    cudaPointerAttributes at;
    if (cudaPointerGetAttributes(&at, p) != cudaSuccess) { (void)cudaGetLastError(); return false; }
    if (at.type == cudaMemoryTypeDevice || at.type == cudaMemoryTypeManaged) return at.device == dev;
    return allow_pinned && at.type == cudaMemoryTypeHost;
}

}  // namespace

extern "C" {

int64_t shine_pool_scratch_bytes(int64_t n_total) {
    if (n_total < 0) return SHINE_ERR_INVALID_ARG;
    return kPoolScratchHeader + 8 * pool_tiles(n_total);
}

int shine_pool_window_append(const shine_sample_pool* pool, const float* coord, const float* label, const float* weight,
                             int64_t n_new, float ox, float oy, float oz, float radius, int64_t* size_out, void* scratch,
                             int64_t scratch_bytes, void* stream) {
    if (!pool || !size_out || !scratch || ((uintptr_t)scratch & 7)) return SHINE_ERR_INVALID_ARG;
    if (pool->size < 0 || pool->capacity < 0 || n_new < 0 || pool->size > pool->capacity) return SHINE_ERR_INVALID_ARG;
    if (n_new > pool->capacity - pool->size) return SHINE_ERR_INVALID_ARG;              // size + n_new > capacity
    if (pool->capacity > 0 && (!pool->coord || !pool->label || !pool->weight)) return SHINE_ERR_INVALID_ARG;
    if (n_new > 0 && (!coord || !label || !weight)) return SHINE_ERR_INVALID_ARG;
    const int64_t total = pool->size + n_new;
    if (scratch_bytes < shine_pool_scratch_bytes(total)) return SHINE_ERR_INVALID_ARG;
    const int dev = device_of(size_out);
    if (dev < 0 || !pointer_usable(scratch, dev, false)) return SHINE_ERR_INVALID_ARG;
    if (pool->capacity > 0 && (!pointer_usable(pool->coord, dev, false) || !pointer_usable(pool->label, dev, false) ||
                               !pointer_usable(pool->weight, dev, false)))
        return SHINE_ERR_INVALID_ARG;
    if (n_new > 0 && (!pointer_usable(coord, dev, true) || !pointer_usable(label, dev, true) ||
                      !pointer_usable(weight, dev, true)))
        return SHINE_ERR_INVALID_ARG;
    const int64_t tiles = pool_tiles(total);
    if (tiles > 0x7fffffff) return SHINE_ERR_UNSUPPORTED;
    DeviceGuard guard(size_out);
    cudaStream_t st = (cudaStream_t)stream;
    if (total == 0) return (int)cudaMemsetAsync(size_out, 0, sizeof(int64_t), st);
    cudaError_t e = cudaMemsetAsync(scratch, 0, (size_t)shine_pool_scratch_bytes(total), st);
    if (e != cudaSuccess) return (int)e;
    PoolArgs a;
    a.coord = pool->coord; a.label = pool->label; a.weight = pool->weight;
    a.new_coord = coord; a.new_label = label; a.new_weight = weight;
    a.size = pool->size; a.n_new = n_new;
    a.ox = ox; a.oy = oy; a.oz = oz; a.r = radius;
    a.tile_counter = reinterpret_cast<unsigned int*>(scratch);
    a.status = reinterpret_cast<unsigned long long*>(static_cast<char*>(scratch) + kPoolScratchHeader);
    a.size_out = size_out;
    pool_window_append_kernel<<<(unsigned)tiles, kPoolThreads, 0, st>>>(a);
    return (int)cudaGetLastError();
}

}  // extern "C"
