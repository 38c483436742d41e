// vex::inclusive_scan / exclusive_scan (vexcl/scan.hpp), vex::inclusive_scan_by_key / exclusive_scan_by_key
// (vexcl/scan_by_key.hpp) and vex::reduce_by_key (vexcl/reduce_by_key.hpp) with the reference's default operators:
// `+` on the values and `==` on the keys.  One reduce-then-scan skeleton serves all five.
//
// Shape rule.  A tile is SCAN_TILE = 4096 elements (256 threads x 16); a slice of n elements has T = ceil(n / 4096)
// tiles, and phases 1 and 3 run one CTA per tile.  Element i is a run head when i == 0 or keys[i] != keys[i - 1]
// (without keys only element 0 is), so a plain scan is a scan by key with one run.  Values are combined as segmented
// pairs (f, s): (fa, sa) . (fb, sb) = (fa | fb, fb ? sb : sa + sb).  Three launches on the caller's stream:
//   reduce  T CTAs; CTA t stages its tile in shared memory, thread j folds its 16 consecutive elements in order
//           (s = head ? x : s + x, from the identity), a Kogge-Stone scan over the 32 lanes of each warp
//           (offsets 1, 2, 4, 8, 16) and one over the 8 warp totals (offsets 1, 2, 4) give the tile's pair; it writes
//           the tile's sum since its last head and its number of heads
//   carry   one CTA of 1024 threads: thread p folds tiles [p P, (p + 1) P), P = ceil(T / 1024), in order, the same
//           Kogge-Stone scans over lanes and the 32 warps give each thread's exclusive prefix, and the thread walks its
//           tiles again writing each tile's carry (the sum since the last head before it) and its first run's number
//   apply   T CTAs; each recomputes its tile's thread prefixes as in reduce, starts thread j at
//           carry + prefix(j), and folds its 16 elements in order; an exclusive scan starts at init + that and restarts
//           at init on every head, writing each value before adding it; reduce_by_key writes only the last element of
//           every run, to okeys[run] and ovals[run]
// Every add is rounded on its own (__dadd_rn, __fadd_rn; integers wrap), and the identity is -0.0 for floats (exact:
// -0.0 + x == x), 0 for integers.  The grid and every add depend on n only, never on the SM count, so results are the
// same bits on every H100 and tests/scan_order.py restates them.  No CTA waits on another: a defect can give a wrong
// answer but not a hang.  A CTA reads all of its tile before it writes it and the carries come from phase 1, so a scan
// in place never reads an element another CTA may have written.
#include "common.cuh"

namespace vexb {
namespace {

constexpr int SCAN_THREADS = 256, SCAN_ITEMS = 16, SCAN_TILE = SCAN_THREADS * SCAN_ITEMS, SCAN_WARPS = SCAN_THREADS / 32;
constexpr int SCAN_CTAS_PER_SM = 3, CARRY_THREADS = 1024, CARRY_WARPS = CARRY_THREADS / 32;
constexpr int SCAN_PADDED = SCAN_TILE + SCAN_TILE / 32;      // one padding word per 32, so blocked reads spread over banks
constexpr unsigned FULL = 0xffffffffu;

enum { KEYS_NONE, KEYS_F32, KEYS_F64, KEYS_B32, KEYS_B64 };
enum { VAL_F64, VAL_F32, VAL_B32, VAL_B64 };
enum { MODE_INCLUSIVE, MODE_EXCLUSIVE, MODE_RBK };

// Keys compare with ==: floats as floats (-0.0 == +0.0, a NaN equals nothing), integers of one width bitwise.
template <int KC> struct key_class { typedef uint32_t word; };
template <> struct key_class<KEYS_F32> {
    typedef uint32_t word;
    static __device__ bool eq(word a, word b) { return __uint_as_float(a) == __uint_as_float(b); }
};
template <> struct key_class<KEYS_F64> {
    typedef uint64_t word;
    static __device__ bool eq(word a, word b) { return __longlong_as_double((long long)a) == __longlong_as_double((long long)b); }
};
template <> struct key_class<KEYS_B32> { typedef uint32_t word; static __device__ bool eq(word a, word b) { return a == b; } };
template <> struct key_class<KEYS_B64> { typedef uint64_t word; static __device__ bool eq(word a, word b) { return a == b; } };

// The add of the element type, rounded on its own; I32 and U32 (I64 and U64) share one wrapping add.
template <int VC> struct val_class;
template <> struct val_class<VAL_F64> {
    typedef double T;
    static __device__ T add(T a, T b) { return __dadd_rn(a, b); }
    static __host__ __device__ T ident() { return -0.0; }
};
template <> struct val_class<VAL_F32> {
    typedef float T;
    static __device__ T add(T a, T b) { return __fadd_rn(a, b); }
    static __host__ __device__ T ident() { return -0.0f; }
};
template <> struct val_class<VAL_B32> {
    typedef uint32_t T;
    static __device__ T add(T a, T b) { return a + b; }
    static __host__ __device__ T ident() { return 0; }
};
template <> struct val_class<VAL_B64> {
    typedef uint64_t T;
    static __device__ T add(T a, T b) { return a + b; }
    static __host__ __device__ T ident() { return 0; }
};

__device__ __forceinline__ int pad(int i) { return i + (i >> 5); }

// Tile elements [tile0, tile0 + tn) of src into r, thread j holding elements 16 j .. 16 j + 15; `fill` past tn.
template <class W>
__device__ __forceinline__ void load_blocked(const W *__restrict__ src, uint32_t tile0, uint32_t tn, W fill,
                                             W (&r)[SCAN_ITEMS], W *sh) {
#pragma unroll
    for (int k = 0; k < SCAN_ITEMS; ++k) {
        const uint32_t i = threadIdx.x + k * SCAN_THREADS;
        sh[pad(i)] = i < tn ? src[tile0 + i] : fill;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < SCAN_ITEMS; ++k) r[k] = sh[pad(threadIdx.x * SCAN_ITEMS + k)];
    __syncthreads();
}

template <class W>
__device__ __forceinline__ void store_blocked(W *__restrict__ dst, uint32_t tile0, uint32_t tn, const W (&r)[SCAN_ITEMS], W *sh) {
#pragma unroll
    for (int k = 0; k < SCAN_ITEMS; ++k) sh[pad(threadIdx.x * SCAN_ITEMS + k)] = r[k];
    __syncthreads();
#pragma unroll
    for (int k = 0; k < SCAN_ITEMS; ++k) {
        const uint32_t i = threadIdx.x + k * SCAN_THREADS;
        if (i < tn) dst[tile0 + i] = sh[pad(i)];
    }
}

// Bit k of the result: element 16 j + k of the tile is a run head.  *ends, bit k: it is the last element of its run.
template <int KC>
__device__ __forceinline__ uint32_t tile_heads(const typename key_class<KC>::word *__restrict__ keys, uint32_t n,
                                               uint32_t tile0, uint32_t tn, void *shv, uint32_t *ends) {
    const uint32_t j0 = threadIdx.x * SCAN_ITEMS;
    if constexpr (KC == KEYS_NONE) {
        *ends = 0;
        return tile0 == 0 && threadIdx.x == 0 ? 1u : 0u;
    } else {
        typedef typename key_class<KC>::word W;
        W *sh = static_cast<W *>(shv);
#pragma unroll
        for (int k = 0; k < SCAN_ITEMS; ++k) {
            const uint32_t i = threadIdx.x + k * SCAN_THREADS;
            sh[pad(i)] = i < tn ? keys[tile0 + i] : 0;
        }
        __syncthreads();
        W prev = j0 == 0 ? (tile0 ? keys[tile0 - 1] : 0) : sh[pad(j0 - 1)];
        uint32_t h = 0;                  // bits 0..16: heads among elements j0 .. j0 + 16
#pragma unroll
        for (int p = 0; p <= SCAN_ITEMS; ++p) {
            const uint32_t g = tile0 + j0 + p;
            if (g < n) {
                const W cur = j0 + p < SCAN_TILE ? sh[pad(j0 + p)] : keys[g];
                if (g == 0 || !key_class<KC>::eq(prev, cur)) h |= 1u << p;
                prev = cur;
            }
        }
        __syncthreads();
        const uint32_t valid = j0 >= tn ? 0u : tn - j0 >= SCAN_ITEMS ? 0xffffu : (1u << (tn - j0)) - 1;
        const uint32_t last = tile0 + j0 < n && n - 1 - tile0 - j0 < SCAN_ITEMS ? 1u << (n - 1 - tile0 - j0) : 0u;
        *ends = ((h >> 1) & valid) | last;
        return h & 0xffffu;
    }
}

template <int VC>
__device__ __forceinline__ void seg_shfl_up(bool &f, typename val_class<VC>::T &s, int o, int lane) {
    const bool fu = __shfl_up_sync(FULL, (int)f, o);
    const typename val_class<VC>::T su = __shfl_up_sync(FULL, s, o);
    if (lane >= o) { s = f ? s : val_class<VC>::add(su, s); f = f || fu; }
}

// Segmented exclusive scan of one pair per thread over a block of NW warps.  (*xf, *xs): the pair of every element
// before this thread, (*af, *as): the block's.  Shared: wf, ws hold NW + 1 entries.
template <int NW, int VC>
__device__ __forceinline__ void block_seg_scan(bool f, typename val_class<VC>::T s, bool *xf, typename val_class<VC>::T *xs,
                                               bool *af, typename val_class<VC>::T *as, int *wf, typename val_class<VC>::T *ws) {
    typedef typename val_class<VC>::T T;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) seg_shfl_up<VC>(f, s, o, lane);
    bool fe = __shfl_up_sync(FULL, (int)f, 1);
    T se = __shfl_up_sync(FULL, s, 1);
    if (lane == 0) { fe = false; se = val_class<VC>::ident(); }
    if (lane == 31) { wf[warp] = f; ws[warp] = s; }
    __syncthreads();
    if (warp == 0) {
        bool g = lane < NW ? wf[lane] != 0 : false;
        T v = lane < NW ? ws[lane] : val_class<VC>::ident();
#pragma unroll
        for (int o = 1; o < NW; o <<= 1) seg_shfl_up<VC>(g, v, o, lane);
        bool pg = __shfl_up_sync(FULL, (int)g, 1);
        T pv = __shfl_up_sync(FULL, v, 1);
        if (lane == 0) { pg = false; pv = val_class<VC>::ident(); }
        __syncwarp();
        if (lane < NW) { wf[lane] = pg; ws[lane] = pv; }
        if (lane == NW - 1) { wf[NW] = g; ws[NW] = v; }
    }
    __syncthreads();
    const bool pf = wf[warp] != 0;
    const T ps = ws[warp];
    *xf = pf || fe;
    *xs = fe ? se : val_class<VC>::add(ps, se);
    *af = wf[NW] != 0;
    *as = ws[NW];
    __syncthreads();
}

// Exclusive sum of one count per thread over a block of NW warps; `wsum` holds NW words.
template <int NW>
__device__ __forceinline__ uint32_t block_count_scan(uint32_t x, uint32_t *wsum, uint32_t *total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t incl = x;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const uint32_t y = __shfl_up_sync(FULL, incl, o); if (lane >= o) incl += y; }
    if (lane == 31) wsum[warp] = incl;
    __syncthreads();
    uint32_t before = 0, all = 0;
#pragma unroll
    for (int w = 0; w < NW; ++w) { const uint32_t c = wsum[w]; before += w < warp ? c : 0; all += c; }
    __syncthreads();
    *total = all;
    return before + incl - x;
}

template <int KC, int VC>
__global__ void __launch_bounds__(SCAN_THREADS, SCAN_CTAS_PER_SM)
scan_reduce_kernel(const typename key_class<KC>::word *__restrict__ keys, const typename val_class<VC>::T *__restrict__ in,
                   uint32_t n, typename val_class<VC>::T *__restrict__ agg, uint32_t *__restrict__ cnt) {
    typedef typename val_class<VC>::T T;
    __shared__ __align__(16) unsigned char sh[SCAN_PADDED * 8];
    __shared__ int wf[SCAN_WARPS + 1];
    __shared__ T ws[SCAN_WARPS + 1];
    __shared__ uint32_t wc[SCAN_WARPS];
    const uint32_t tile0 = blockIdx.x * SCAN_TILE, tn = min((uint32_t)SCAN_TILE, n - tile0);
    uint32_t ends;
    const uint32_t heads = tile_heads<KC>(keys, n, tile0, tn, sh, &ends);
    T x[SCAN_ITEMS];
    load_blocked(in, tile0, tn, val_class<VC>::ident(), x, reinterpret_cast<T *>(sh));
    bool f = false;
    T s = val_class<VC>::ident();
#pragma unroll
    for (int k = 0; k < SCAN_ITEMS; ++k) {
        if (heads >> k & 1) { f = true; s = x[k]; } else s = val_class<VC>::add(s, x[k]);
    }
    bool xf, af;
    T xs, as;
    block_seg_scan<SCAN_WARPS, VC>(f, s, &xf, &xs, &af, &as, wf, ws);
    uint32_t total;
    block_count_scan<SCAN_WARPS>(__popc(heads), wc, &total);
    if (threadIdx.x == 0) { agg[blockIdx.x] = as; cnt[blockIdx.x] = total; }
}

// One CTA: agg[t] (tile sums since their last head) -> carry into tile t; cnt[t] (heads in tile t) -> heads before
// tile t; cnt[T] = all heads.
template <int VC>
__global__ void __launch_bounds__(CARRY_THREADS)
scan_carry_kernel(typename val_class<VC>::T *__restrict__ agg, uint32_t *__restrict__ cnt, uint32_t ntiles) {
    typedef typename val_class<VC>::T T;
    __shared__ int wf[CARRY_WARPS + 1];
    __shared__ T ws[CARRY_WARPS + 1];
    __shared__ uint32_t wc[CARRY_WARPS];
    const uint32_t per = (ntiles + CARRY_THREADS - 1) / CARRY_THREADS;
    const uint32_t lo = min(ntiles, threadIdx.x * per), hi = min(ntiles, lo + per);
    bool f = false;
    T s = val_class<VC>::ident();
    uint32_t c = 0;
    for (uint32_t t = lo; t < hi; ++t) {
        const uint32_t ct = cnt[t];
        const T a = agg[t];
        if (ct) { f = true; s = a; } else s = val_class<VC>::add(s, a);
        c += ct;
    }
    bool xf, af;
    T xs, as;
    block_seg_scan<CARRY_WARPS, VC>(f, s, &xf, &xs, &af, &as, wf, ws);
    uint32_t total;
    uint32_t base = block_count_scan<CARRY_WARPS>(c, wc, &total);
    T run = xs;
    for (uint32_t t = lo; t < hi; ++t) {
        const uint32_t ct = cnt[t];
        const T a = agg[t];
        agg[t] = run;
        cnt[t] = base;
        run = ct ? a : val_class<VC>::add(run, a);
        base += ct;
    }
    if (threadIdx.x == 0) cnt[ntiles] = total;
}

template <int KC, int VC, int MODE>
__global__ void __launch_bounds__(SCAN_THREADS, SCAN_CTAS_PER_SM)
scan_apply_kernel(const typename key_class<KC>::word *__restrict__ keys, const typename val_class<VC>::T *in,
                  typename val_class<VC>::T *out, uint32_t n, const typename val_class<VC>::T *__restrict__ carry,
                  const uint32_t *__restrict__ base, typename val_class<VC>::T init,
                  typename key_class<KC>::word *__restrict__ okeys) {
    typedef typename val_class<VC>::T T;
    __shared__ __align__(16) unsigned char sh[SCAN_PADDED * 8];
    __shared__ int wf[SCAN_WARPS + 1];
    __shared__ T ws[SCAN_WARPS + 1];
    __shared__ uint32_t wc[SCAN_WARPS];
    const uint32_t tile0 = blockIdx.x * SCAN_TILE, tn = min((uint32_t)SCAN_TILE, n - tile0);
    uint32_t ends;
    const uint32_t heads = tile_heads<KC>(keys, n, tile0, tn, sh, &ends);
    T x[SCAN_ITEMS];
    load_blocked(in, tile0, tn, val_class<VC>::ident(), x, reinterpret_cast<T *>(sh));
    bool f = false;
    T s = val_class<VC>::ident();
#pragma unroll
    for (int k = 0; k < SCAN_ITEMS; ++k) {
        if (heads >> k & 1) { f = true; s = x[k]; } else s = val_class<VC>::add(s, x[k]);
    }
    bool xf, af;
    T xs, as;
    block_seg_scan<SCAN_WARPS, VC>(f, s, &xf, &xs, &af, &as, wf, ws);
    T r = xf ? xs : val_class<VC>::add(carry[blockIdx.x], xs);
    if constexpr (MODE == MODE_INCLUSIVE) {
#pragma unroll
        for (int k = 0; k < SCAN_ITEMS; ++k) { r = heads >> k & 1 ? x[k] : val_class<VC>::add(r, x[k]); x[k] = r; }
        store_blocked(out, tile0, tn, x, reinterpret_cast<T *>(sh));
    } else if constexpr (MODE == MODE_EXCLUSIVE) {
        r = val_class<VC>::add(init, r);
#pragma unroll
        for (int k = 0; k < SCAN_ITEMS; ++k) {
            if (heads >> k & 1) r = init;
            const T o = r;
            r = val_class<VC>::add(r, x[k]);
            x[k] = o;
        }
        store_blocked(out, tile0, tn, x, reinterpret_cast<T *>(sh));
    } else {
        uint32_t total;
        uint32_t run = base[blockIdx.x] + block_count_scan<SCAN_WARPS>(__popc(heads), wc, &total);
        const uint32_t g0 = tile0 + threadIdx.x * SCAN_ITEMS;
#pragma unroll
        for (int k = 0; k < SCAN_ITEMS; ++k) {
            r = heads >> k & 1 ? x[k] : val_class<VC>::add(r, x[k]);
            run += heads >> k & 1;
            if (ends >> k & 1) { out[run - 1] = r; okeys[run - 1] = keys[g0 + k]; }
        }
    }
}

size_t align256(size_t b) { return (b + 255) / 256 * 256; }
size_t scan_tiles(size_t n) { return (n + SCAN_TILE - 1) / SCAN_TILE; }

// Workspace: one value per tile (sums, then carries) and T + 1 counts (heads, then run numbers, then their total).
size_t workspace_bytes(size_t n, size_t vb) {
    if (n == 0) return 0;
    const size_t t = scan_tiles(n);
    return align256(t * vb) + align256((t + 1) * 4);
}

bool valid_dtype(int dt) { return dt >= VEXB_F64 && dt <= VEXB_U64; }

int key_class_of(int dt) {
    switch (dt) {
        case -1: return KEYS_NONE;
        case VEXB_F32: return KEYS_F32;
        case VEXB_F64: return KEYS_F64;
        case VEXB_I32: case VEXB_U32: return KEYS_B32;
        default: return KEYS_B64;
    }
}

int val_class_of(int dt) {
    switch (dt) {
        case VEXB_F64: return VAL_F64;
        case VEXB_F32: return VAL_F32;
        case VEXB_I32: case VEXB_U32: return VAL_B32;
        default: return VAL_B64;
    }
}

struct scan_args {
    const void *keys, *in;
    void *out, *okeys;
    uint32_t n;
    const void *init;      // host, one element; NULL: zero
    void *ws;
};

// Phases 1 and 2 (reduce, carry) if `reduce`, then phase 3 (apply) in `mode` if `apply`.
template <int KC, int VC>
int run_scan(cudaStream_t s, const scan_args &a, int mode, bool apply, bool reduce) {
    typedef typename val_class<VC>::T T;
    typedef typename key_class<KC>::word W;
    const uint32_t ntiles = (uint32_t)scan_tiles(a.n);
    T *agg = static_cast<T *>(a.ws);
    uint32_t *cnt = reinterpret_cast<uint32_t *>(static_cast<char *>(a.ws) + align256(ntiles * sizeof(T)));
    const W *keys = static_cast<const W *>(a.keys);
    const T *in = static_cast<const T *>(a.in);
    if (reduce) {
        scan_reduce_kernel<KC, VC><<<ntiles, SCAN_THREADS, 0, s>>>(keys, in, a.n, agg, cnt);
        VEXB_LAUNCHED();
        scan_carry_kernel<VC><<<1, CARRY_THREADS, 0, s>>>(agg, cnt, ntiles);
        VEXB_LAUNCHED();
    }
    if (!apply) return VEXB_OK;
    T init = T();
    if (a.init) std::memcpy(&init, a.init, sizeof(T));
    T *out = static_cast<T *>(a.out);
    if (mode == MODE_INCLUSIVE)
        scan_apply_kernel<KC, VC, MODE_INCLUSIVE><<<ntiles, SCAN_THREADS, 0, s>>>(keys, in, out, a.n, agg, cnt, init, nullptr);
    else if (mode == MODE_EXCLUSIVE)
        scan_apply_kernel<KC, VC, MODE_EXCLUSIVE><<<ntiles, SCAN_THREADS, 0, s>>>(keys, in, out, a.n, agg, cnt, init, nullptr);
    else if constexpr (KC != KEYS_NONE)
        scan_apply_kernel<KC, VC, MODE_RBK><<<ntiles, SCAN_THREADS, 0, s>>>(keys, in, out, a.n, agg, cnt, init,
                                                                           static_cast<W *>(a.okeys));
    VEXB_LAUNCHED();
    return VEXB_OK;
}

template <int KC>
int run_scan_vals(cudaStream_t s, int val_dtype, const scan_args &a, int mode, bool apply, bool reduce) {
    switch (val_class_of(val_dtype)) {
        case VAL_F64: return run_scan<KC, VAL_F64>(s, a, mode, apply, reduce);
        case VAL_F32: return run_scan<KC, VAL_F32>(s, a, mode, apply, reduce);
        case VAL_B32: return run_scan<KC, VAL_B32>(s, a, mode, apply, reduce);
        default:      return run_scan<KC, VAL_B64>(s, a, mode, apply, reduce);
    }
}

int dispatch(int dev, void *stream, int key_dtype, int val_dtype, const scan_args &a, int mode, bool apply, bool reduce) {
    DeviceGuard g(dev);
    if (!g.ok) VEXB_FAIL(VEXB_ERR_CUDA, "cudaSetDevice(%d) failed", dev);
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    switch (key_class_of(key_dtype)) {
        case KEYS_NONE: return run_scan_vals<KEYS_NONE>(s, val_dtype, a, mode, apply, reduce);
        case KEYS_F32:  return run_scan_vals<KEYS_F32>(s, val_dtype, a, mode, apply, reduce);
        case KEYS_F64:  return run_scan_vals<KEYS_F64>(s, val_dtype, a, mode, apply, reduce);
        case KEYS_B32:  return run_scan_vals<KEYS_B32>(s, val_dtype, a, mode, apply, reduce);
        default:        return run_scan_vals<KEYS_B64>(s, val_dtype, a, mode, apply, reduce);
    }
}

} // namespace
} // namespace vexb

using namespace vexb;

#define SCAN_CHECK_COMMON(n, val_dtype, ws, wsb)                                                                     \
    VEXB_CHECK(n <= (size_t)INT32_MAX, "%zu elements: a slice scans at most 2^31 - 1", n);                           \
    do {                                                                                                             \
        const size_t need_ = workspace_bytes(n, dtype_size(val_dtype));                                              \
        VEXB_CHECK(need_ == 0 || ws, "d_workspace is NULL (%zu bytes needed)", need_);                               \
        VEXB_CHECK(wsb >= need_, "workspace too small (%zu < %zu bytes)", wsb, need_);                               \
    } while (0)

extern "C" int vexb_scan_workspace_bytes(size_t n, int val_dtype, size_t *bytes) {
    VEXB_CHECK(valid_dtype(val_dtype), "unknown value dtype %d", val_dtype);
    VEXB_CHECK(bytes, "bytes is NULL");
    *bytes = workspace_bytes(n, dtype_size(val_dtype));
    return VEXB_OK;
}

extern "C" int vexb_scan(int dev, void *stream, const void *in, void *out, int dtype, size_t n, int exclusive,
                         const void *h_init, void *d_workspace, size_t workspace_bytes_) {
    VEXB_CHECK(valid_dtype(dtype), "unknown value dtype %d", dtype);
    VEXB_CHECK(n == 0 || (in && out), "NULL input or output for %zu elements", n);
    SCAN_CHECK_COMMON(n, dtype, d_workspace, workspace_bytes_);
    if (n == 0) return VEXB_OK;
    const scan_args a{nullptr, in, out, nullptr, (uint32_t)n, h_init, d_workspace};
    return dispatch(dev, stream, -1, dtype, a, exclusive ? MODE_EXCLUSIVE : MODE_INCLUSIVE, true, true);
}

extern "C" int vexb_scan_by_key(int dev, void *stream, const void *keys, int key_dtype, const void *ivals, void *ovals,
                                int val_dtype, size_t n, int exclusive, const void *h_init, void *d_workspace,
                                size_t workspace_bytes_) {
    VEXB_CHECK(valid_dtype(key_dtype), "unknown key dtype %d", key_dtype);
    VEXB_CHECK(valid_dtype(val_dtype), "unknown value dtype %d", val_dtype);
    VEXB_CHECK(n == 0 || (keys && ivals && ovals), "NULL keys, input or output for %zu elements", n);
    VEXB_CHECK(n == 0 || keys != ovals, "keys and ovals are the same buffer");
    SCAN_CHECK_COMMON(n, val_dtype, d_workspace, workspace_bytes_);
    if (n == 0) return VEXB_OK;
    const scan_args a{keys, ivals, ovals, nullptr, (uint32_t)n, h_init, d_workspace};
    return dispatch(dev, stream, key_dtype, val_dtype, a, exclusive ? MODE_EXCLUSIVE : MODE_INCLUSIVE, true, true);
}

extern "C" int vexb_reduce_by_key_count(int dev, void *stream, const void *ikeys, int key_dtype, const void *ivals,
                                        int val_dtype, size_t n, void *d_workspace, size_t workspace_bytes_,
                                        size_t *nruns) {
    VEXB_CHECK(valid_dtype(key_dtype), "unknown key dtype %d", key_dtype);
    VEXB_CHECK(valid_dtype(val_dtype), "unknown value dtype %d", val_dtype);
    VEXB_CHECK(n == 0 || (ikeys && ivals), "NULL keys or values for %zu elements", n);
    VEXB_CHECK(nruns, "nruns is NULL");
    SCAN_CHECK_COMMON(n, val_dtype, d_workspace, workspace_bytes_);
    *nruns = 0;
    if (n == 0) return VEXB_OK;
    const scan_args a{ikeys, ivals, nullptr, nullptr, (uint32_t)n, nullptr, d_workspace};
    VEXB_TRY(dispatch(dev, stream, key_dtype, val_dtype, a, MODE_RBK, false, true));
    DeviceGuard g(dev);
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    uint32_t total = 0;
    const uint32_t *cnt = reinterpret_cast<const uint32_t *>(static_cast<const char *>(d_workspace) +
                                                             align256(scan_tiles(n) * dtype_size(val_dtype)));
    VEXB_CUDA(cudaMemcpyAsync(&total, cnt + scan_tiles(n), sizeof(total), cudaMemcpyDeviceToHost, s));
    VEXB_CUDA(cudaStreamSynchronize(s));
    *nruns = total;
    return VEXB_OK;
}

extern "C" int vexb_reduce_by_key_write(int dev, void *stream, const void *ikeys, int key_dtype, const void *ivals,
                                        int val_dtype, size_t n, void *okeys, void *ovals, void *d_workspace,
                                        size_t workspace_bytes_) {
    VEXB_CHECK(valid_dtype(key_dtype), "unknown key dtype %d", key_dtype);
    VEXB_CHECK(valid_dtype(val_dtype), "unknown value dtype %d", val_dtype);
    VEXB_CHECK(n == 0 || (ikeys && ivals && okeys && ovals), "NULL keys or values for %zu elements", n);
    VEXB_CHECK(n == 0 || (okeys != ikeys && okeys != ivals && ovals != ikeys && ovals != ivals && okeys != ovals),
               "okeys and ovals must be buffers apart from each other and from ikeys and ivals");
    SCAN_CHECK_COMMON(n, val_dtype, d_workspace, workspace_bytes_);
    if (n == 0) return VEXB_OK;
    const scan_args a{ikeys, ivals, ovals, okeys, (uint32_t)n, nullptr, d_workspace};
    return dispatch(dev, stream, key_dtype, val_dtype, a, MODE_RBK, true, false);
}
