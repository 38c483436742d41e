// vex::sort / vex::sort_by_key for the built-in comparators (vexcl/sort.hpp:2120-2182): a stable LSD radix sort of one
// device slice, and the stable host merge of sorted slices (sort.hpp:2070-2116 merges them on the host too).
//
// Shape rule.  A tile is SORT_TILE = 4096 elements (256 threads x 16).  A slice of n elements has T = ceil(n / 4096)
// tiles and is cut into G = min(T, 2 x SMs) runs of consecutive tiles, run b holding tiles [b T / G, (b + 1) T / G).
// Every pass takes 8 bits of the ordered key (csrc/sort_keys.cuh), lowest first: 4 passes for 4-byte keys, 8 for
// 8-byte keys, alternating between the caller's buffers and the workspace, so the result lands in the caller's buffers.
// One pass is three launches on the caller's stream:
//   count    G CTAs; CTA b counts the digits of its run into column b of a digit-major 256 x G table
//   scan     one CTA turns the table into exclusive offsets: where digit d of run b starts in the output
//   scatter  G CTAs; CTA b walks its run tile by tile, ranks each element among the equal digits of the tile in input
//            order (warp match + per-warp counters + a prefix across warps), stages the tile in shared memory grouped
//            by digit and writes it out, so consecutive threads write consecutive addresses of one digit's run
// No CTA waits on another; each pass's result depends only on its input, so the output is deterministic.
#include "common.cuh"
#include "sort_keys.cuh"
#include <vector>

namespace vexb {
namespace {

constexpr int SORT_THREADS = 256, SORT_ITEMS = 16, SORT_TILE = SORT_THREADS * SORT_ITEMS;
constexpr int SORT_WARPS = SORT_THREADS / 32, SORT_CTAS_PER_SM = 2, SORT_SCAN_THREADS = 1024;
constexpr unsigned FULL = 0xffffffffu;

template <int DT> using bits_t = typename sort_bits<DT>::type;
template <int VB> struct payload { typedef uint32_t type; };
template <> struct payload<8> { typedef uint64_t type; };

// Exclusive scan of one value per thread across a block of NW warps; `wsum` holds NW words of shared memory.
template <int NW>
__device__ __forceinline__ uint32_t block_exclusive_scan(uint32_t x, uint32_t *wsum) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t incl = x;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const uint32_t y = __shfl_up_sync(FULL, incl, o); if (lane >= o) incl += y; }
    if (lane == 31) wsum[warp] = incl;
    __syncthreads();
    if (warp == 0) {
        const uint32_t w = lane < NW ? wsum[lane] : 0;
        uint32_t wi = w;
#pragma unroll
        for (int o = 1; o < NW; o <<= 1) { const uint32_t y = __shfl_up_sync(FULL, wi, o); if (lane >= o) wi += y; }
        if (lane < NW) wsum[lane] = wi - w;
    }
    __syncthreads();
    const uint32_t r = wsum[warp] + incl - x;
    __syncthreads();
    return r;
}

__device__ __forceinline__ void run_of(uint32_t ntiles, uint32_t *t0, uint32_t *t1) {
    *t0 = (uint32_t)((uint64_t)blockIdx.x * ntiles / gridDim.x);
    *t1 = (uint32_t)((uint64_t)(blockIdx.x + 1) * ntiles / gridDim.x);
}

template <int DT>
__global__ void __launch_bounds__(SORT_THREADS, SORT_CTAS_PER_SM)
sort_count_kernel(const bits_t<DT> *__restrict__ keys, uint32_t n, bits_t<DT> desc_mask, int shift, uint32_t ntiles,
                  uint32_t *__restrict__ table) {
    __shared__ uint32_t hist[256];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    hist[threadIdx.x] = 0;
    __syncthreads();
    uint32_t t0, t1;
    run_of(ntiles, &t0, &t1);
    for (uint32_t t = t0; t < t1; ++t) {
        const uint32_t base = t * SORT_TILE + warp * (32 * SORT_ITEMS) + lane;
        bits_t<DT> k[SORT_ITEMS];
#pragma unroll
        for (int j = 0; j < SORT_ITEMS; ++j) k[j] = base + 32 * j < n ? keys[base + 32 * j] : 0;
#pragma unroll
        for (int j = 0; j < SORT_ITEMS; ++j) {
            const bool valid = base + 32 * j < n;
            const uint32_t d = valid ? (uint32_t)(sort_order<DT>(k[j], desc_mask) >> shift) & 0xff : 256;
            const unsigned peers = __match_any_sync(FULL, d);
            if (valid && lane == __ffs(peers) - 1) atomicAdd(&hist[d], __popc(peers));
        }
    }
    __syncthreads();
    table[threadIdx.x * gridDim.x + blockIdx.x] = hist[threadIdx.x];
}

// One CTA: table[0 .. len) (digit-major counts) -> exclusive prefix sums in place.
__global__ void __launch_bounds__(SORT_SCAN_THREADS) sort_scan_kernel(uint32_t *__restrict__ table, uint32_t len) {
    __shared__ uint32_t wsum[SORT_SCAN_THREADS / 32];
    const uint32_t per = (len + SORT_SCAN_THREADS - 1) / SORT_SCAN_THREADS;
    const uint32_t lo = min(len, threadIdx.x * per), hi = min(len, lo + per);
    uint32_t sum = 0;
    for (uint32_t i = lo; i < hi; ++i) sum += table[i];
    uint32_t run = block_exclusive_scan<SORT_SCAN_THREADS / 32>(sum, wsum);
    for (uint32_t i = lo; i < hi; ++i) { const uint32_t c = table[i]; table[i] = run; run += c; }
}

template <int DT, int VB>
__global__ void __launch_bounds__(SORT_THREADS, SORT_CTAS_PER_SM)
sort_scatter_kernel(const bits_t<DT> *__restrict__ kin, bits_t<DT> *__restrict__ kout,
                    const typename payload<VB>::type *__restrict__ vin, typename payload<VB>::type *__restrict__ vout,
                    uint32_t n, bits_t<DT> desc_mask, int shift, uint32_t ntiles, const uint32_t *__restrict__ table) {
    typedef bits_t<DT> K;
    typedef typename payload<VB>::type V;
    extern __shared__ __align__(16) unsigned char smem[];
    K *skeys = reinterpret_cast<K *>(smem);
    V *svals = reinterpret_cast<V *>(smem + SORT_TILE * sizeof(K));
    __shared__ uint32_t warp_count[SORT_WARPS][256];    // per warp and digit: count, then the warp's start in the digit
    __shared__ uint32_t tile_start[256];                 // where digit d starts in the staged tile
    __shared__ uint32_t out_base[256];                   // output index of staged element i with digit d: out_base[d] + i
    __shared__ uint32_t wsum[SORT_WARPS];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const unsigned lanes_below = (1u << lane) - 1;
    uint32_t running = table[threadIdx.x * gridDim.x + blockIdx.x];   // next output index of digit threadIdx.x
    uint32_t t0, t1;
    run_of(ntiles, &t0, &t1);
    for (uint32_t t = t0; t < t1; ++t) {
#pragma unroll
        for (int w = 0; w < SORT_WARPS; ++w) warp_count[w][threadIdx.x] = 0;
        const uint32_t tile0 = t * SORT_TILE, tile_n = min((uint32_t)SORT_TILE, n - tile0);
        const uint32_t base = tile0 + warp * (32 * SORT_ITEMS) + lane;
        K k[SORT_ITEMS];
        V v[VB ? SORT_ITEMS : 1];
        uint32_t slot[SORT_ITEMS];          // digit << 16 | rank of the element among its digit in the warp
#pragma unroll
        for (int j = 0; j < SORT_ITEMS; ++j) {
            const bool valid = base + 32 * j < n;
            k[j] = valid ? kin[base + 32 * j] : 0;
            if constexpr (VB != 0) v[j] = valid ? vin[base + 32 * j] : 0;
        }
        __syncthreads();
        // A warp's elements are base + 32 j: item j of lane l precedes item j of lane l + 1 and item j + 1 of any lane,
        // so ranking items in j order, lanes in order within an item, ranks them in input order.
#pragma unroll
        for (int j = 0; j < SORT_ITEMS; ++j) {
            const bool valid = base + 32 * j < n;
            const uint32_t d = valid ? (uint32_t)(sort_order<DT>(k[j], desc_mask) >> shift) & 0xff : 256;
            const unsigned peers = __match_any_sync(FULL, d);
            const int leader = __ffs(peers) - 1;
            uint32_t before = 0;
            if (valid && lane == leader) { before = warp_count[warp][d]; warp_count[warp][d] = before + __popc(peers); }
            before = __shfl_sync(FULL, before, leader);
            slot[j] = d << 16 | (before + __popc(peers & lanes_below));
            __syncwarp();
        }
        __syncthreads();
        uint32_t count = 0;
#pragma unroll
        for (int w = 0; w < SORT_WARPS; ++w) { const uint32_t c = warp_count[w][threadIdx.x]; warp_count[w][threadIdx.x] = count; count += c; }
        const uint32_t start = block_exclusive_scan<SORT_WARPS>(count, wsum);
        tile_start[threadIdx.x] = start;
        out_base[threadIdx.x] = running - start;
        running += count;
        __syncthreads();
#pragma unroll
        for (int j = 0; j < SORT_ITEMS; ++j) {
            const uint32_t d = slot[j] >> 16;
            if (d < 256) {
                const uint32_t pos = tile_start[d] + warp_count[warp][d] + (slot[j] & 0xffff);
                skeys[pos] = k[j];
                if constexpr (VB != 0) svals[pos] = v[j];
            }
        }
        __syncthreads();
        for (uint32_t i = threadIdx.x; i < tile_n; i += SORT_THREADS) {
            const K key = skeys[i];
            const uint32_t o = out_base[(uint32_t)(sort_order<DT>(key, desc_mask) >> shift) & 0xff] + i;
            kout[o] = key;
            if constexpr (VB != 0) vout[o] = svals[i];
        }
        __syncthreads();
    }
}

size_t align256(size_t b) { return (b + 255) / 256 * 256; }
size_t sort_tiles(size_t n) { return (n + SORT_TILE - 1) / SORT_TILE; }

// Workspace: a second key buffer, a second value buffer, and the 256 x G table (G <= number of tiles).
size_t workspace_bytes(size_t n, size_t kb, size_t vb) {
    if (n < 2) return 0;
    return align256(n * kb) + align256(n * vb) + align256(256 * 4 * sort_tiles(n));
}

template <int DT, int VB>
int sort_slice(int dev, cudaStream_t s, void *keys, void *vals, uint32_t n, bool descending, void *ws) {
    typedef bits_t<DT> K;
    typedef typename payload<VB>::type V;
    const uint32_t ntiles = (uint32_t)sort_tiles(n);
    const uint32_t G = (uint32_t)std::min<size_t>(ntiles, (size_t)SORT_CTAS_PER_SM * sm_count(dev));
    const K mask = descending ? ~K(0) : K(0);
    char *w = static_cast<char *>(ws);
    K *kbuf[2] = {static_cast<K *>(keys), reinterpret_cast<K *>(w)};
    V *vbuf[2] = {static_cast<V *>(vals), reinterpret_cast<V *>(w + align256((size_t)n * sizeof(K)))};
    uint32_t *table = reinterpret_cast<uint32_t *>(w + align256((size_t)n * sizeof(K)) + align256((size_t)n * VB));
    const int smem = SORT_TILE * (int)(sizeof(K) + VB);
    VEXB_CUDA(cudaFuncSetAttribute(sort_scatter_kernel<DT, VB>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    for (int pass = 0; pass < (int)sizeof(K); ++pass) {
        const int src = pass & 1, shift = 8 * pass;
        sort_count_kernel<DT><<<G, SORT_THREADS, 0, s>>>(kbuf[src], n, mask, shift, ntiles, table);
        VEXB_LAUNCHED();
        sort_scan_kernel<<<1, SORT_SCAN_THREADS, 0, s>>>(table, 256 * G);
        VEXB_LAUNCHED();
        sort_scatter_kernel<DT, VB><<<G, SORT_THREADS, smem, s>>>(kbuf[src], kbuf[src ^ 1], vbuf[src], vbuf[src ^ 1], n, mask,
                                                                  shift, ntiles, table);
        VEXB_LAUNCHED();
    }
    return VEXB_OK;
}

template <int DT>
int sort_slice_vals(int dev, cudaStream_t s, void *keys, void *vals, size_t vb, uint32_t n, bool descending, void *ws) {
    switch (vb) {
        case 0: return sort_slice<DT, 0>(dev, s, keys, vals, n, descending, ws);
        case 4: return sort_slice<DT, 4>(dev, s, keys, vals, n, descending, ws);
        default: return sort_slice<DT, 8>(dev, s, keys, vals, n, descending, ws);
    }
}

bool valid_dtype(int dt) { return dt >= VEXB_F64 && dt <= VEXB_U64; }

// Stable k-way merge of sorted runs: the smallest ordered key goes first, the lowest part on ties.
template <int DT>
void merge_parts(int nparts, const size_t *part, const void *keys, const void *vals, size_t vb, bool descending,
                 void *keys_out, void *vals_out) {
    typedef bits_t<DT> K;
    const K mask = descending ? ~K(0) : K(0);
    const K *k = static_cast<const K *>(keys);
    K *ko = static_cast<K *>(keys_out);
    std::vector<size_t> pos(part, part + nparts);
    const size_t n = part[nparts];
    for (size_t o = 0; o < n; ++o) {
        int best = -1;
        K best_key = 0;
        for (int p = 0; p < nparts; ++p) {
            if (pos[p] == part[p + 1]) continue;
            const K key = sort_order<DT>(k[pos[p]], mask);
            if (best < 0 || key < best_key) { best = p; best_key = key; }
        }
        const size_t i = pos[best]++;
        ko[o] = k[i];
        if (vb) std::memcpy(static_cast<char *>(vals_out) + o * vb, static_cast<const char *>(vals) + i * vb, vb);
    }
}

} // namespace
} // namespace vexb

using namespace vexb;

extern "C" int vexb_sort_workspace_bytes(size_t n, int key_dtype, int val_dtype, size_t *bytes) {
    VEXB_CHECK(valid_dtype(key_dtype), "unknown key dtype %d", key_dtype);
    VEXB_CHECK(val_dtype == -1 || valid_dtype(val_dtype), "unknown value dtype %d (-1: keys only)", val_dtype);
    VEXB_CHECK(bytes, "bytes is NULL");
    *bytes = workspace_bytes(n, dtype_size(key_dtype), val_dtype < 0 ? 0 : dtype_size(val_dtype));
    return VEXB_OK;
}

extern "C" int vexb_sort(int dev, void *stream, void *keys, int key_dtype, void *vals, int val_dtype, size_t n,
                         int descending, void *d_workspace, size_t workspace_bytes_) {
    VEXB_CHECK(valid_dtype(key_dtype), "unknown key dtype %d", key_dtype);
    VEXB_CHECK(val_dtype == -1 || valid_dtype(val_dtype), "unknown value dtype %d (-1: keys only)", val_dtype);
    VEXB_CHECK(keys || n == 0, "keys is NULL for %zu elements", n);
    VEXB_CHECK(!vals || val_dtype >= 0, "vals is given without a val_dtype");
    VEXB_CHECK(vals || val_dtype < 0 || n == 0, "val_dtype %d is given without vals", val_dtype);
    VEXB_CHECK(!vals || vals != keys, "vals and keys are the same buffer");
    VEXB_CHECK(n <= (size_t)INT32_MAX, "%zu elements: a slice sorts at most 2^31 - 1", n);
    const size_t vb = val_dtype < 0 ? 0 : dtype_size(val_dtype);
    const size_t need = workspace_bytes(n, dtype_size(key_dtype), vb);
    VEXB_CHECK(need == 0 || d_workspace, "d_workspace is NULL (%zu bytes needed)", need);
    VEXB_CHECK(workspace_bytes_ >= need, "workspace too small (%zu < %zu bytes)", workspace_bytes_, need);
    if (n < 2) return VEXB_OK;
    DeviceGuard g(dev);
    if (!g.ok) VEXB_FAIL(VEXB_ERR_CUDA, "cudaSetDevice(%d) failed", dev);
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const uint32_t m = (uint32_t)n;
    const bool desc = descending != 0;
    switch (key_dtype) {
        case VEXB_F64: return sort_slice_vals<VEXB_F64>(dev, s, keys, vals, vb, m, desc, d_workspace);
        case VEXB_F32: return sort_slice_vals<VEXB_F32>(dev, s, keys, vals, vb, m, desc, d_workspace);
        case VEXB_I32: return sort_slice_vals<VEXB_I32>(dev, s, keys, vals, vb, m, desc, d_workspace);
        case VEXB_U32: return sort_slice_vals<VEXB_U32>(dev, s, keys, vals, vb, m, desc, d_workspace);
        case VEXB_I64: return sort_slice_vals<VEXB_I64>(dev, s, keys, vals, vb, m, desc, d_workspace);
        default:       return sort_slice_vals<VEXB_U64>(dev, s, keys, vals, vb, m, desc, d_workspace);
    }
}

extern "C" int vexb_sort_merge(int nparts, const size_t *part, const void *keys, int key_dtype, const void *vals,
                               int val_dtype, int descending, void *keys_out, void *vals_out) {
    VEXB_CHECK(nparts >= 1 && part, "bad part offsets");
    VEXB_CHECK(valid_dtype(key_dtype), "unknown key dtype %d", key_dtype);
    VEXB_CHECK(val_dtype == -1 || valid_dtype(val_dtype), "unknown value dtype %d (-1: keys only)", val_dtype);
    for (int p = 0; p < nparts; ++p) VEXB_CHECK(part[p] <= part[p + 1], "part offsets decrease at part %d", p);
    const size_t n = part[nparts] - part[0];
    VEXB_CHECK(n == 0 || (keys && keys_out), "NULL keys");
    VEXB_CHECK(val_dtype < 0 || n == 0 || (vals && vals_out), "NULL values with val_dtype %d", val_dtype);
    VEXB_CHECK(val_dtype >= 0 || (!vals && !vals_out), "values are given without a val_dtype");
    if (n == 0) return VEXB_OK;
    // offsets relative to the first part, so `keys` may point at the first element of part 0
    std::vector<size_t> rel(nparts + 1);
    for (int p = 0; p <= nparts; ++p) rel[p] = part[p] - part[0];
    const size_t vb = val_dtype < 0 ? 0 : dtype_size(val_dtype);
    const bool desc = descending != 0;
    switch (key_dtype) {
        case VEXB_F64: merge_parts<VEXB_F64>(nparts, rel.data(), keys, vals, vb, desc, keys_out, vals_out); break;
        case VEXB_F32: merge_parts<VEXB_F32>(nparts, rel.data(), keys, vals, vb, desc, keys_out, vals_out); break;
        case VEXB_I32: merge_parts<VEXB_I32>(nparts, rel.data(), keys, vals, vb, desc, keys_out, vals_out); break;
        case VEXB_U32: merge_parts<VEXB_U32>(nparts, rel.data(), keys, vals, vb, desc, keys_out, vals_out); break;
        case VEXB_I64: merge_parts<VEXB_I64>(nparts, rel.data(), keys, vals, vb, desc, keys_out, vals_out); break;
        default:       merge_parts<VEXB_U64>(nparts, rel.data(), keys, vals, vb, desc, keys_out, vals_out); break;
    }
    return VEXB_OK;
}
