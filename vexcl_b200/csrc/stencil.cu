// vex::stencil<T> convolution (vexcl/stencil.hpp:168-330; semantics as the reference benchmark's CPU check,
// examples/benchmark.cpp:318-327):
//     y[i] (=|+=) alpha * sum_{k < width} s[k] * X(i + k - center),     X(j) = x[clamp(j, 0, n-1)] over the WHOLE vector.
// One device slice per call; positions left of the slice come from `left` (the `center` elements before it) and
// positions right of it from `right` (the `width-1-center` elements after it) when the slice is not at an end of the
// vector, otherwise they clamp to the slice's first / last element.
//
// Design.  16 B/element of compulsory traffic (x once, y once; +8 for `+=`) against 2*width FP64 instructions
// (products and sums are rounded separately, in tap order, like the reference loop): at width 21 the two are about
// balanced, so neither shared memory nor issue slots may cost more than that.  Hence
//   * a block stages its x window (1024 outputs + width-1 neighbours) and the taps in shared memory once;
//   * a thread owns EIGHT CONSECUTIVE outputs and slides a 16-element register window over the taps in chunks of 8:
//     per chunk 8 window loads + 8 tap loads (broadcast) feed 64 multiply-adds, 4x fewer shared-memory reads per
//     product than one-output-per-thread;
//   * the window is stored with one pad word per 8 elements, so the stride-8 accesses of neighbouring lanes fall in
//     different banks (stride 9);
//   * a thread's 8 results leave as 32-byte chunks, each two 128-bit stores (and `+=` reads y the same way).
#include <algorithm>
#include <atomic>
#include <mutex>
#include <string>
#include <vector>
#include "common.cuh"
#include "shapes.cuh"
#include "jit.hpp"

namespace vexb {
namespace {

constexpr int ST_THREADS = 128;
constexpr int ST_E = 8;                                  // consecutive outputs per thread
constexpr int ST_B = ST_THREADS * ST_E;                  // outputs per block

__host__ __device__ __forceinline__ int st_pad(int p) { return p + (p >> 3); }
__host__ __device__ __forceinline__ int st_ceil8(int w) { return (w + 7) & ~7; }

template <class T>
__global__ void __launch_bounds__(ST_THREADS) stencil_kernel(const T *__restrict__ s, int width, int center,
                                                             const T *__restrict__ x, long long n,
                                                             const T *__restrict__ left, const T *__restrict__ right,
                                                             T *y, T alpha, int append, int vec_io) {
    typedef Arith<T> A;
    extern __shared__ __align__(16) unsigned char st_smem[];
    const int wlen = ST_B + st_ceil8(width);             // window positions staged (those past ST_B+width-2 are never used in a product)
    T *win = reinterpret_cast<T *>(st_smem);
    T *taps = win + st_pad(wlen) + 1;
    const long long b0 = (long long)blockIdx.x * ST_B;
    const int rhalo = width - 1 - center;

    // ---- stage the window: position p holds X(b0 - center + p) --------------------------------------------------
    // Eight loads per thread are issued before the first store (addresses selected without branches: end clamps and
    // halo buffers are pointer selects).  A load -> store loop would leave one load in flight per thread and stall on
    // those stores.
    auto source = [&](int p) -> const T * {
        const long long j = b0 - center + p;
        if (j < 0) return left ? left + (center + j) : x;
        if (j >= n) {
            const long long r = j - n;
            return (right && rhalo > 0) ? right + (r < rhalo ? r : rhalo - 1) : x + (n - 1);
        }
        return x + j;
    };
    // Tiles whose whole window lies inside the slice (all but the first and last few) load x directly: no clamps, no
    // pointer selects -- the kernel is issue-bound, so every instruction outside the multiply-adds counts.
    const bool inside = b0 - center >= 0 && b0 - center + (long long)wlen <= n;
    for (int p0 = threadIdx.x; p0 < wlen; p0 += 8 * ST_THREADS) {
        T v[8];
        if (inside) {
            const T *src = x + (b0 - center) + p0;
#pragma unroll
            for (int u = 0; u < 8; ++u) v[u] = src[p0 + u * ST_THREADS < wlen ? u * ST_THREADS : 0];
        } else {
#pragma unroll
            for (int u = 0; u < 8; ++u) { const int p = p0 + u * ST_THREADS; v[u] = *source(p < wlen ? p : wlen - 1); }
        }
#pragma unroll
        for (int u = 0; u < 8; ++u) { const int p = p0 + u * ST_THREADS; if (p < wlen) win[st_pad(p)] = v[u]; }
    }
    for (int k = threadIdx.x; k < st_ceil8(width); k += ST_THREADS) taps[k] = k < width ? s[k] : T(0);
    __syncthreads();

    const int o = threadIdx.x * ST_E;                     // first output of this thread within the block
    if (b0 + o >= n) return;
    T sum[ST_E], lo[8], hi[8];
#pragma unroll
    for (int e = 0; e < ST_E; ++e) sum[e] = T(0);
#pragma unroll
    for (int j = 0; j < 8; ++j) lo[j] = win[st_pad(o + j)];
    const T *wp = win + st_pad(o) + 9;                    // st_pad(o + 8 + c) = st_pad(o) + 9 + c + (c >> 3) for o a multiple of 8
    int kk = 0;
    for (; kk + 8 <= width; kk += 8) {                    // full chunks of 8 taps: straight-line, no per-tap test
        T sk[8];
        const T *wq = wp + kk + (kk >> 3);
#pragma unroll
        for (int j = 0; j < 8; ++j) { hi[j] = wq[j]; sk[j] = taps[kk + j]; }
#pragma unroll
        for (int j = 0; j < 8; ++j) {
#pragma unroll
            for (int e = 0; e < ST_E; ++e) sum[e] = A::add(sum[e], A::mul(sk[j], (e + j < 8) ? lo[e + j] : hi[e + j - 8]));
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) lo[j] = hi[j];
    }
    if (kk < width) {                                     // the last 1..7 taps (block-uniform)
        const int rem = width - kk;
        T sk[8];
        const T *wq = wp + kk + (kk >> 3);
#pragma unroll
        for (int j = 0; j < 8; ++j) { hi[j] = wq[j]; sk[j] = taps[kk + j]; }
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            if (j < rem) {
#pragma unroll
                for (int e = 0; e < ST_E; ++e) sum[e] = A::add(sum[e], A::mul(sk[j], (e + j < 8) ? lo[e + j] : hi[e + j - 8]));
            }
        }
    }

    // ---- y (=|+=) alpha * sum -------------------------------------------------------------------------------------
    const long long i0 = b0 + o;
    constexpr int PER = Lanes<T>::E;                      // elements per 32-byte chunk: 4 doubles, 8 floats
    if (vec_io && i0 + ST_E <= n) {
#pragma unroll
        for (int q = 0; q < ST_E / PER; ++q) {
            Vec256 out = {};
            if (append) {
                const Vec256 old = ldg256(y + i0 + q * PER);
#pragma unroll
                for (int e = 0; e < PER; ++e) Lanes<T>::set(out, e, A::add(Lanes<T>::get(old, e), A::mul(alpha, sum[q * PER + e])));
            } else {
#pragma unroll
                for (int e = 0; e < PER; ++e) Lanes<T>::set(out, e, A::mul(alpha, sum[q * PER + e]));
            }
            stg256(y + i0 + q * PER, out);
        }
    } else {
#pragma unroll
        for (int e = 0; e < ST_E; ++e) {
            if (i0 + e < n) { const T v = A::mul(alpha, sum[e]); y[i0 + e] = append ? A::add(y[i0 + e], v) : v; }
        }
    }
}

// ---- pipelined version: persistent blocks, the next window arrives while this one is multiplied ------------------
// Same arithmetic and layout as stencil_kernel.  A block walks the tiles b, b + grid, ...; the window of its NEXT tile is
// copied global -> shared asynchronously (cp.async, 8 bytes per element straight into the padded layout, no registers)
// while the FP64 phase of the current tile runs from the other buffer.  With one-shot blocks the HBM stream and the FP64
// pipe only overlap across the blocks of an SM.
template <class T> __device__ __forceinline__ void cp_async_elem(T *dst_smem, const T *src) {
    const uint32_t d = (uint32_t)__cvta_generic_to_shared(dst_smem);
    if (sizeof(T) == 8) asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" :: "r"(d), "l"(src) : "memory");
    else                asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" :: "r"(d), "l"(src) : "memory");
}

template <class T>
__global__ void __launch_bounds__(ST_THREADS) stencil_pipe_kernel(const T *__restrict__ s, int width, int center,
                                                                  const T *__restrict__ x, long long n,
                                                                  const T *__restrict__ left, const T *__restrict__ right,
                                                                  T *y, T alpha, int append, int vec_io, long long tiles) {
    typedef Arith<T> A;
    extern __shared__ __align__(16) unsigned char st_smem[];
    const int wlen = ST_B + st_ceil8(width);
    const int wpad = st_pad(wlen) + 1;
    T *winbuf = reinterpret_cast<T *>(st_smem);           // two windows
    T *taps = winbuf + 2 * wpad;
    const int rhalo = width - 1 - center;

    auto fetch = [&](long long tile, T *win) {
        const long long b0 = tile * ST_B;
        for (int p = threadIdx.x; p < wlen; p += ST_THREADS) {
            const long long j = b0 - center + p;
            const T *src;
            if (j < 0) src = left ? left + (center + j) : x;
            else if (j >= n) { const long long r = j - n; src = (right && rhalo > 0) ? right + (r < rhalo ? r : rhalo - 1) : x + (n - 1); }
            else src = x + j;
            cp_async_elem<T>(win + st_pad(p), src);
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
    };

    long long tile = blockIdx.x;
    if (tile >= tiles) return;
    fetch(tile, winbuf);
    for (int k = threadIdx.x; k < st_ceil8(width); k += ST_THREADS) taps[k] = k < width ? s[k] : T(0);
    int buf = 0;
    for (; tile < tiles; tile += gridDim.x, buf ^= 1) {
        asm volatile("cp.async.wait_all;" ::: "memory");
        __syncthreads();                                  // this tile's window is complete; nobody reads the other buffer any more
        const long long next = tile + gridDim.x;
        if (next < tiles) fetch(next, winbuf + (buf ^ 1) * wpad);
        const T *win = winbuf + buf * wpad;
        const long long b0 = tile * ST_B;
        const int o = threadIdx.x * ST_E;
        if (b0 + o >= n) continue;
        T sum[ST_E], lo[8], hi[8];
#pragma unroll
        for (int e = 0; e < ST_E; ++e) sum[e] = T(0);
#pragma unroll
        for (int j = 0; j < 8; ++j) lo[j] = win[st_pad(o + j)];
        for (int kk = 0; kk < width; kk += 8) {
            const int rem = width - kk;
            T sk[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) { hi[j] = win[st_pad(o + kk + 8 + j)]; sk[j] = taps[kk + j]; }
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                if (j < rem) {
#pragma unroll
                    for (int e = 0; e < ST_E; ++e) sum[e] = A::add(sum[e], A::mul(sk[j], (e + j < 8) ? lo[e + j] : hi[e + j - 8]));
                }
            }
#pragma unroll
            for (int j = 0; j < 8; ++j) lo[j] = hi[j];
        }
        const long long i0 = b0 + o;
        constexpr int PER = Lanes<T>::E;
        if (vec_io && i0 + ST_E <= n) {
#pragma unroll
            for (int q = 0; q < ST_E / PER; ++q) {
                Vec256 out = {};
                if (append) {
                    const Vec256 old = ldg256(y + i0 + q * PER);
#pragma unroll
                    for (int e = 0; e < PER; ++e) Lanes<T>::set(out, e, A::add(Lanes<T>::get(old, e), A::mul(alpha, sum[q * PER + e])));
                } else {
#pragma unroll
                    for (int e = 0; e < PER; ++e) Lanes<T>::set(out, e, A::mul(alpha, sum[q * PER + e]));
                }
                stg256(y + i0 + q * PER, out);
            }
        } else {
#pragma unroll
            for (int e = 0; e < ST_E; ++e) {
                if (i0 + e < n) { const T v = A::mul(alpha, sum[e]); y[i0 + e] = append ? A::add(y[i0 + e], v) : v; }
            }
        }
    }
}

template <class T>
static int stencil_launch(int dev, cudaStream_t st, const T *s, int width, int center, const T *x, size_t n,
                          const T *left, const T *right, T *y, T alpha, int append) {
    const int wlen = ST_B + st_ceil8(width);
    const size_t smem = ((size_t)st_pad(wlen) + 1 + st_ceil8(width)) * sizeof(T);
    if (smem > 200 * 1024) VEXB_FAIL(VEXB_ERR_UNSUPPORTED, "stencil of %d taps does not fit in shared memory", width);
    static std::atomic<unsigned long long> attr_set[2];
    const int ti = sizeof(T) == 8 ? 0 : 1;
    const unsigned long long bit = 1ull << (dev & 63);
    if (smem > 48 * 1024 && !(attr_set[ti].load() & bit)) {
        VEXB_CUDA(cudaFuncSetAttribute(stencil_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
        attr_set[ti].fetch_or(bit);
    }
    const unsigned blocks = (unsigned)((n + ST_B - 1) / ST_B);
    const int vec_io = aligned32(y) ? 1 : 0;
    // stencil.kernel: 1 = one block per tile (default), 0 = pipelined persistent blocks -- its 8-byte cp.async copies into
    // the padded layout cost issue slots that the overlap across the resident blocks of an SM already makes up for
    // (H100 SXM, width 21, N = 2^26: 0.451 ms one block per tile against 0.50 ms pipelined)
    const size_t smem2 = (2 * ((size_t)st_pad(wlen) + 1) + st_ceil8(width)) * sizeof(T);
    if (param("stencil.kernel", 1) == 0 && smem2 <= 100 * 1024) {
        static std::atomic<unsigned long long> attr2[2];
        if (smem2 > 48 * 1024 && !(attr2[ti].load() & bit)) {
            VEXB_CUDA(cudaFuncSetAttribute(stencil_pipe_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024));
            attr2[ti].fetch_or(bit);
        }
        int per_sm = 0;
        VEXB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, stencil_pipe_kernel<T>, ST_THREADS, smem2));
        const long cap = param("stencil.blocks_per_sm", 0);
        if (cap > 0 && per_sm > cap) per_sm = (int)cap;
        const size_t resident = (size_t)std::max(per_sm, 1) * (size_t)sm_count(dev);
        if ((size_t)blocks > resident) {
            stencil_pipe_kernel<T><<<(unsigned)resident, ST_THREADS, smem2, st>>>(s, width, center, x, (long long)n, left, right, y, alpha, append,
                                                                              vec_io, (long long)blocks);
            VEXB_LAUNCHED();
            return VEXB_OK;
        }
    }
    stencil_kernel<T><<<blocks, ST_THREADS, smem, st>>>(s, width, center, x, (long long)n, left, right, y, alpha, append, vec_io);
    VEXB_LAUNCHED();
    return VEXB_OK;
}

} // namespace
} // namespace vexb

using namespace vexb;

extern "C" int vexb_stencil_apply(int dev, void *stream, int dtype, const void *s, int width, int center,
                                  const void *x, size_t n, const void *left, const void *right,
                                  void *y, double alpha, int append) {
    VEXB_CHECK(dtype == VEXB_F64 || dtype == VEXB_F32, "stencil values must be float or double");
    VEXB_CHECK(width >= 1 && center >= 0 && center < width, "stencil needs width >= 1 and 0 <= center < width");
    if (!n) return VEXB_OK;
    VEXB_CHECK(s && x && y, "null pointer");
    VEXB_CHECK(n < ((size_t)1 << 40), "slice too long");
    DeviceGuard g(dev); VEXB_CHECK(g.ok, "cannot select device %d", dev);
    cudaStream_t st = (cudaStream_t)stream;
    if (dtype == VEXB_F64)
        return stencil_launch<double>(dev, st, (const double *)s, width, center, (const double *)x, n, (const double *)left,
                                      (const double *)right, (double *)y, alpha, append);
    return stencil_launch<float>(dev, st, (const float *)s, width, center, (const float *)x, n, (const float *)left,
                                 (const float *)right, (float *)y, (float)alpha, append);
}

extern "C" int vexb_copy_peer(int dst_dev, void *dst, int src_dev, const void *src, size_t bytes, void *stream) {
    if (!bytes) return VEXB_OK;
    VEXB_CHECK(dst && src, "null pointer");
    DeviceGuard g(dst_dev); VEXB_CHECK(g.ok, "cannot select device %d", dst_dev);
    if (dst_dev == src_dev) VEXB_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
    else VEXB_CUDA(cudaMemcpyPeerAsync(dst, dst_dev, src, src_dev, bytes, (cudaStream_t)stream));
    return VEXB_OK;
}

// ---- user-defined stencil operators (VEX_STENCIL_OPERATOR, vexcl/stencil.hpp:510-680) -----------------------------------
// y[i] (=|+=) alpha * f(X), where the body of f is C source supplied at run time and X[k] is the element k places from
// i (clamped at the ends of the vector, halos as above).  Like the reference, the kernel is generated per operator:
// a block stages its window in shared memory and hands the body a pointer into it, so `X[-1]`, `X[0]`, `X[1]` are
// plain shared-memory reads.  Compiled by NVRTC at first use (--fmad=false), cached per (operator, device).
namespace vexb {
namespace {
struct StencilOp { int dtype, width, center; std::string body; };
std::mutex g_somx;
std::vector<StencilOp> g_sops;

std::string stencil_op_source(const StencilOp &op) {
    const char *T = op.dtype == VEXB_F64 ? "double" : "float";
    std::string s;
    s += "// generated by libvexb200 (csrc/stencil.cu): user-defined stencil operator\n";
    s += std::string("typedef ") + T + " T;\n";
    s += "#define WIDTH " + std::to_string(op.width) + "\n#define CENTER " + std::to_string(op.center) + "\n";
    s += "#define RHALO (WIDTH - 1 - CENTER)\n";
    s += "__device__ __forceinline__ T stencil_oper(const T *X) {\n" + op.body + "\n}\n";
    s += "extern \"C\" __global__ void __launch_bounds__(256) vexb_stencil_op(const T *__restrict__ x, long long n,\n"
         "        const T *__restrict__ left, const T *__restrict__ right, T *y, T alpha, int append) {\n"
         "    __shared__ T win[256 + WIDTH - 1];\n"
         "    const long long b0 = (long long)blockIdx.x * 256;\n"
         "    for (int p = threadIdx.x; p < 256 + WIDTH - 1; p += 256) {\n"
         "        const long long j = b0 - CENTER + p;\n"
         "        T v;\n"
         "        if (j < 0) v = left ? left[CENTER + j] : x[0];\n"
         "        else if (j >= n) { const long long r = j - n; v = (right && RHALO > 0) ? right[r < RHALO ? r : RHALO - 1] : x[n - 1]; }\n"
         "        else v = x[j];\n"
         "        win[p] = v;\n"
         "    }\n"
         "    __syncthreads();\n"
         "    const long long i = b0 + threadIdx.x;\n"
         "    if (i >= n) return;\n"
         "    const T v = alpha * stencil_oper(win + CENTER + threadIdx.x);\n"
         "    y[i] = append ? y[i] + v : v;\n"
         "}\n";
    return s;
}
} // namespace
} // namespace vexb

extern "C" int vexb_stencil_operator_register(int dtype, int width, int center, const char *body, int *id) {
    VEXB_CHECK(id && body, "null argument");
    VEXB_CHECK(dtype == VEXB_F64 || dtype == VEXB_F32, "stencil operators work on float or double");
    VEXB_CHECK(width >= 1 && width <= 4096 && center >= 0 && center < width, "stencil operator needs 1 <= width <= 4096 and 0 <= center < width");
    std::lock_guard<std::mutex> lock(vexb::g_somx);
    for (size_t k = 0; k < vexb::g_sops.size(); ++k) {
        const auto &o = vexb::g_sops[k];
        if (o.dtype == dtype && o.width == width && o.center == center && o.body == body) { *id = (int)k; return VEXB_OK; }
    }
    vexb::g_sops.push_back({dtype, width, center, body});
    *id = (int)vexb::g_sops.size() - 1;
    return VEXB_OK;
}

extern "C" int vexb_stencil_operator_source(int id, char *buf, size_t *len, int compile) {
    VEXB_CHECK(len, "len is NULL");
    std::string src;
    {
        std::lock_guard<std::mutex> lock(vexb::g_somx);
        VEXB_CHECK(id >= 0 && (size_t)id < vexb::g_sops.size(), "unknown stencil operator %d", id);
        src = vexb::stencil_op_source(vexb::g_sops[(size_t)id]);
    }
    return vexb::jit_print(std::move(src), compile, false, buf, len);
}

extern "C" int vexb_stencil_operator_apply(int dev, void *stream, int id, const void *x, size_t n, const void *left,
                                           const void *right, void *y, double alpha, int append) {
    vexb::StencilOp op;
    {
        std::lock_guard<std::mutex> lock(vexb::g_somx);
        VEXB_CHECK(id >= 0 && (size_t)id < vexb::g_sops.size(), "unknown stencil operator %d", id);
        op = vexb::g_sops[(size_t)id];
    }
    if (!n) return VEXB_OK;
    VEXB_CHECK(x && y, "null pointer");
    VEXB_CHECK(n < ((size_t)1 << 38), "slice too long");
    DeviceGuard g(dev); VEXB_CHECK(g.ok, "cannot select device %d", dev);
    void *fn = nullptr;
    // the operator's body is user text: the device's program header goes first
    VEXB_TRY(vexb::jit_program(dev, "stencil:" + std::to_string(id), "vexb_stencil_op", vexb::program_header(dev), [&](vexb::JitBuild *b) {
        b->text = vexb::stencil_op_source(op);
        return VEXB_OK;
    }, true, &fn));
    long long nn = (long long)n;
    double a64 = alpha; float a32 = (float)alpha;
    void *args[] = {&x, &nn, &left, &right, &y, op.dtype == VEXB_F64 ? (void *)&a64 : (void *)&a32, &append};
    return vexb::jit_launch(fn, (unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream, args);
}
