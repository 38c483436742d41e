// Block and complex sparse strips on one device: y (=|+=) alpha * A * x with B x B blocks (B = 2, 3, 4) or complex numbers
// as values, the products of vex::sparse::{csr, ell, matrix}<std::array<std::array<T,B>,B>> (the reference's custom value
// types, sparse/distributed.hpp:17-21 rhs_of + sparse/spmv_ops.hpp spmv_ops_impl) and of vex::sparse::{csr, ell,
// matrix}<std::complex<T>> (the spmv_ops_impl of the reference's examples/complex_spmv.cpp).
//
// Layout: sliced ELL (SELL-32-sigma, as VEXB_FMT_SELL) over BLOCK rows, from the same host sell_layout, sigma
// ("spmv.sell_sigma") and perm / slice_ptr.  One int32 block column per slot (-1 = padding).  Values are planar per
// slot: component c = r*B + q of slot k, lane l of slice s sits at val[(slice_ptr[s] + 32k) * B*B + 32c + l], so every
// value load of a warp is 32 consecutive T whatever B is.  One column and one gather of B consecutive x values serve
// B*B values: 8B^2 + 4 bytes per stored block in double against 12B^2 for the same block expanded into scalar CSR.
// Complex strips are the same layout over rows with 2 components per slot, c = 0 (re) and c = 1 (im): 2 sizeof(T) + 4
// bytes per stored entry, and one 2 sizeof(T)-byte gather of x (re, im) per slot.
// User strips (vex::sparse::{csr, ell, matrix}<V> for a user type V with a vex::sparse::spmv_ops_impl<V, X>) are the same
// layout over rows with ONE opaque component of val_bytes per slot: lane l of slot k in slice s holds the value at index
// slice_ptr[s] + 32k + l, so a warp's value loads are 32 consecutive V.  Their kernel is generated from the user's source
// snippets and compiled by NVRTC at first use (usr_source below).
#include "hostlogic.hpp"
#include "jit.hpp"
#include "spmv_dev.cuh"
#include <map>
#include <mutex>
#include <sstream>
#include <vector>

namespace vexb {
// Device arrays of a sliced-ELL strip with planar values, shared by block and complex strips.
struct sell_strip {
    int *slice_ptr = nullptr, *perm = nullptr, *col = nullptr; void *val = nullptr;
    size_t n_slices = 0, n_slots = 0, device_bytes = 0;
};
}

struct vexb_bspmat : vexb::sell_strip {
    int dev = 0, block = 0, val_dtype = VEXB_F64;
    size_t nrows = 0, ncols = 0, nnzb = 0;     // block rows, block columns, stored blocks
};

struct vexb_zspmat : vexb::sell_strip {
    int dev = 0, val_dtype = VEXB_F64;         // VEXB_F64: std::complex<double>, VEXB_F32: std::complex<float>
    size_t nrows = 0, ncols = 0, nnz = 0;      // rows, columns, stored complex entries
};

struct vexb_usrmat : vexb::sell_strip {
    int dev = 0, val_bytes = 0;                // sizeof(V)
    size_t nrows = 0, ncols = 0, nnz = 0;      // rows, columns, stored values
};

namespace vexb {

// Slots in flight per loop turn: U * (B*B values + 1 column + B gathers) loads per lane.  Picked so that no
// instantiation spills (-Xptxas -v, DESIGN.md section 3 lists the register counts).
template <class T, int B> constexpr int bsell_unroll() { return B == 2 ? 4 : 2; }

// y_r += the block row's blocks in storage order; inside a block, row r is t = a_r0 x_0, t = t + a_r1 x_1, ..., then
// s_r = s_r + t, every product and sum rounded on its own (the order of the reference test's loop and of its
// append_product, tests/sparse_matrices.cpp:271-281).
template <class T, int B, int U>
__device__ __forceinline__ void bsell_slots(const int *cp, const T *vp, int k, const T *__restrict__ x,
                                            uint64_t stream, uint64_t keep, T (&sum)[B]) {
    int c[U]; T v[U][B * B], xv[U][B];
#pragma unroll
    for (int u = 0; u < U; ++u) {
        c[u] = ldg_stream(cp + (size_t)(k + u) * 32, stream);
#pragma unroll
        for (int e = 0; e < B * B; ++e) v[u][e] = ldg_stream(vp + (size_t)(k + u) * 32 * (B * B) + 32 * e, stream);
    }
#pragma unroll
    for (int u = 0; u < U; ++u)
#pragma unroll
        for (int q = 0; q < B; ++q) xv[u][q] = c[u] != -1 ? ldg_keep(x + (size_t)c[u] * B + q, keep) : T(0);
#pragma unroll
    for (int u = 0; u < U; ++u) {
        if (c[u] == -1) continue;
#pragma unroll
        for (int r = 0; r < B; ++r) {
            T t = t_mul<T>(v[u][r * B], xv[u][0]);
#pragma unroll
            for (int q = 1; q < B; ++q) t = t_add<T>(t, t_mul<T>(v[u][r * B + q], xv[u][q]));
            sum[r] = t_add<T>(sum[r], t);
        }
    }
}

// One warp per slice, one lane per block row, B partial sums in registers.
template <class T, int B>
__global__ void __launch_bounds__(256) bsell_kernel(size_t n_slices, const int *__restrict__ slice_ptr, const int *__restrict__ perm,
                                                    const int *__restrict__ col, const T *__restrict__ val,
                                                    const T *__restrict__ x, T *y, T alpha, int append) {
    constexpr int U = bsell_unroll<T, B>();
    const size_t s = (size_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (s >= n_slices) return;
    const int lane = threadIdx.x & 31;
    const uint64_t stream = l2_policy_stream(), keep = l2_policy_keep();
    const int base = __ldg(slice_ptr + s), w = (__ldg(slice_ptr + s + 1) - base) >> 5;
    const int r = ldg_stream(perm + s * 32 + lane, stream);
    const int *cp = col + base + lane;
    const T *vp = val + (size_t)base * (B * B) + lane;      // 64-bit: slots * B*B passes 2^31 long before the slot count
    T sum[B];
#pragma unroll
    for (int q = 0; q < B; ++q) sum[q] = T(0);
    int k = 0;
    for (; k + U <= w; k += U) bsell_slots<T, B, U>(cp, vp, k, x, stream, keep, sum);
    for (; k < w; ++k) bsell_slots<T, B, 1>(cp, vp, k, x, stream, keep, sum);
    if (r >= 0)
#pragma unroll
        for (int q = 0; q < B; ++q) store_y<T>(y, (size_t)r * B + q, sum[q], alpha, append);
}

template <class T>
static int bspmv_launch(const vexb_bspmat *A, cudaStream_t st, const T *x, T *y, T alpha, int append) {
    if (A->nrows == 0) return VEXB_OK;
    if (A->nnzb == 0) {
        // as vexb_spmv on an empty strip: y = A*x zeroes y, y += A*x leaves it alone
        if (!append) VEXB_CUDA(cudaMemsetAsync(y, 0, A->nrows * A->block * sizeof(T), st));
        return VEXB_OK;
    }
    const unsigned grid = (unsigned)((A->n_slices + 7) / 8);
    switch (A->block) {
        case 2: bsell_kernel<T, 2><<<grid, 256, 0, st>>>(A->n_slices, A->slice_ptr, A->perm, A->col, (const T *)A->val, x, y, alpha, append); break;
        case 3: bsell_kernel<T, 3><<<grid, 256, 0, st>>>(A->n_slices, A->slice_ptr, A->perm, A->col, (const T *)A->val, x, y, alpha, append); break;
        default: bsell_kernel<T, 4><<<grid, 256, 0, st>>>(A->n_slices, A->slice_ptr, A->perm, A->col, (const T *)A->val, x, y, alpha, append); break;
    }
    VEXB_LAUNCHED();
    return VEXB_OK;
}

template <class T> struct complex_of;
template <> struct complex_of<double> { typedef double2 type; };
template <> struct complex_of<float> { typedef float2 type; };

// Slots in flight per loop turn: U * (2 values + 1 column) streaming loads and U gathers of x per lane.  No spills in
// either precision (-Xptxas -v, DESIGN.md section 3 lists the register counts).
constexpr int kZsellUnroll = 4;

// The row's entries a + bi in storage order (the spmv_ops_impl of the reference's examples/complex_spmv.cpp):
// s_re = s_re + (a xr - b xi), s_im = s_im + (a xi + b xr), every product and sum rounded on its own.
template <class T, int U>
__device__ __forceinline__ void zsell_slots(const int *cp, const T *vp, int k, const typename complex_of<T>::type *__restrict__ x,
                                            uint64_t stream, uint64_t keep, T &re, T &im) {
    typedef typename complex_of<T>::type C2;
    int c[U]; T a[U], b[U]; C2 xv[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
        c[u] = ldg_stream(cp + (size_t)(k + u) * 32, stream);
        a[u] = ldg_stream(vp + (size_t)(k + u) * 64, stream);
        b[u] = ldg_stream(vp + (size_t)(k + u) * 64 + 32, stream);
    }
#pragma unroll
    for (int u = 0; u < U; ++u) xv[u] = c[u] != -1 ? ldg_keep(x + c[u], keep) : C2{T(0), T(0)};
#pragma unroll
    for (int u = 0; u < U; ++u) {
        if (c[u] == -1) continue;
        re = t_add<T>(re, t_sub<T>(t_mul<T>(a[u], xv[u].x), t_mul<T>(b[u], xv[u].y)));
        im = t_add<T>(im, t_add<T>(t_mul<T>(a[u], xv[u].y), t_mul<T>(b[u], xv[u].x)));
    }
}

// One warp per slice, one lane per row, the real and imaginary sums in registers.
template <class T>
__global__ void __launch_bounds__(256) zsell_kernel(size_t n_slices, const int *__restrict__ slice_ptr, const int *__restrict__ perm,
                                                    const int *__restrict__ col, const T *__restrict__ val,
                                                    const typename complex_of<T>::type *__restrict__ x, T *y, T alpha, int append) {
    constexpr int U = kZsellUnroll;
    const size_t s = (size_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (s >= n_slices) return;
    const int lane = threadIdx.x & 31;
    const uint64_t stream = l2_policy_stream(), keep = l2_policy_keep();
    const int base = __ldg(slice_ptr + s), w = (__ldg(slice_ptr + s + 1) - base) >> 5;
    const int r = ldg_stream(perm + s * 32 + lane, stream);
    const int *cp = col + base + lane;
    const T *vp = val + (size_t)base * 2 + lane;
    T re = T(0), im = T(0);
    int k = 0;
    for (; k + U <= w; k += U) zsell_slots<T, U>(cp, vp, k, x, stream, keep, re, im);
    for (; k < w; ++k) zsell_slots<T, 1>(cp, vp, k, x, stream, keep, re, im);
    if (r >= 0) {
        store_y<T>(y, (size_t)r * 2, re, alpha, append);
        store_y<T>(y, (size_t)r * 2 + 1, im, alpha, append);
    }
}

template <class T>
static int zspmv_launch(const vexb_zspmat *A, cudaStream_t st, const T *x, T *y, T alpha, int append) {
    if (A->nrows == 0) return VEXB_OK;
    if (A->nnz == 0) {
        if (!append) VEXB_CUDA(cudaMemsetAsync(y, 0, A->nrows * 2 * sizeof(T), st));
        return VEXB_OK;
    }
    const unsigned grid = (unsigned)((A->n_slices + 7) / 8);
    zsell_kernel<T><<<grid, 256, 0, st>>>(A->n_slices, A->slice_ptr, A->perm, A->col, (const T *)A->val,
                                          (const typename complex_of<T>::type *)x, y, alpha, append);
    VEXB_LAUNCHED();
    return VEXB_OK;
}

template <class E>
static int upload_array(const std::vector<E> &h, void **d, size_t *bytes_acc) {
    *d = nullptr;
    if (h.empty()) return VEXB_OK;
    VEXB_CUDA(cudaMalloc(d, h.size() * sizeof(E)));
    VEXB_CUDA(cudaMemcpy(*d, h.data(), h.size() * sizeof(E), cudaMemcpyHostToDevice));
    *bytes_acc += h.size() * sizeof(E);
    return VEXB_OK;
}

// Host form of a strip whose arguments passed sell_check: row pointers from 0, columns, and the sliced-ELL layout.
struct sell_host {
    std::vector<int> rp, col, perm, sptr;
    size_t nnz = 0, slots = 0;
};

// The argument checks of vexb_bsr_create, vexb_zsr_create and vexb_usr_create but the value type's; none touches a device.  `unit` is "block " when rows,
// columns and entries count blocks, "" otherwise.
static int sell_check(size_t nrows, size_t ncols, const void *ptr, int ptr_bytes, const void *col, int col_bytes,
                      const void *val, const char *unit, sell_host &h) {
    VEXB_CHECK(ptr_bytes == 4 || ptr_bytes == 8, "ptr_bytes must be 4 or 8");
    VEXB_CHECK(col_bytes == 4 || col_bytes == 8, "col_bytes must be 4 or 8");
    VEXB_CHECK(nrows == 0 || ptr, "ptr is NULL");
    VEXB_CHECK(nrows < (size_t)INT32_MAX && ncols < (size_t)INT32_MAX, "%sdimensions exceed 32-bit local indices", unit);
    const int64_t p0 = nrows ? read_index(ptr, ptr_bytes, 0) : 0;
    const int64_t nnz = nrows ? read_index(ptr, ptr_bytes, nrows) - p0 : 0;
    VEXB_CHECK(nnz >= 0 && nnz < (int64_t)INT32_MAX - 64, "%lld stored %sentries do not fit 32-bit row pointers", (long long)nnz, unit);
    VEXB_CHECK(nnz == 0 || (col && val), "col/val is NULL");
    h.nnz = (size_t)nnz;
    h.rp.assign(nrows + 1, 0);
    h.col.resize((size_t)nnz);
    for (size_t i = 1; i <= nrows; ++i) {
        const int64_t v = read_index(ptr, ptr_bytes, i) - p0;
        VEXB_CHECK(v >= h.rp[i - 1] && v <= nnz, "row pointers decrease at %srow %zu", unit, i);
        h.rp[i] = (int)v;
    }
    for (size_t j = 0; j < (size_t)nnz; ++j) {
        const int64_t cj = read_index(col, col_bytes, j);
        VEXB_CHECK(cj >= 0 && (size_t)cj < ncols, "%scolumn %lld out of range at entry %zu", unit, (long long)cj, j);
        h.col[j] = (int)cj;
    }
    VEXB_CHECK(sell_layout(nrows, h.rp.data(), param("spmv.sell_sigma", 1024), h.perm, h.sptr, &h.slots),
               "%sstrip too large for 32-bit slot offsets", unit);
    return VEXB_OK;
}

// Host packing of the planar slots (see the top of this file), `comps` components of `comp_bytes` bytes per stored entry;
// padding slots keep column -1 and zero bytes.
static int sell_upload(sell_strip *S, const sell_host &h, const void *val, size_t comp_bytes, size_t comps) {
    S->n_slices = h.sptr.size() - 1; S->n_slots = h.slots;
    std::vector<int> scol(S->n_slots, -1);
    std::vector<unsigned char> sval(S->n_slots * comps * comp_bytes, 0);
    const unsigned char *src = static_cast<const unsigned char *>(val);
    for (size_t sl = 0; sl < S->n_slices; ++sl)
        for (int l = 0; l < 32; ++l) {
            const int r = h.perm[sl * 32 + l];
            if (r < 0) continue;
            for (int j = h.rp[r], k = 0; j < h.rp[r + 1]; ++j, ++k) {
                const size_t slot = (size_t)h.sptr[sl] + (size_t)k * 32;
                scol[slot + l] = h.col[j];
                for (size_t c = 0; c < comps; ++c)
                    memcpy(&sval[(slot * comps + 32 * c + l) * comp_bytes], src + ((size_t)j * comps + c) * comp_bytes, comp_bytes);
            }
        }
    VEXB_TRY(upload_array(h.sptr, (void **)&S->slice_ptr, &S->device_bytes));
    VEXB_TRY(upload_array(h.perm, (void **)&S->perm, &S->device_bytes));
    VEXB_TRY(upload_array(scol, (void **)&S->col, &S->device_bytes));
    VEXB_TRY(upload_array(sval, &S->val, &S->device_bytes));
    // cudaMemcpy from pageable memory may return before its DMA has landed, and the products run on non-blocking streams,
    // which do not wait for the legacy stream: without this, a product launched right after create() can read a tail of
    // values that is not there yet
    VEXB_CUDA(cudaStreamSynchronize(0));
    return VEXB_OK;
}

static void sell_free(sell_strip *S) {
    cudaFree(S->slice_ptr); cudaFree(S->perm); cudaFree(S->col); cudaFree(S->val);
}

} // namespace vexb

using namespace vexb;

extern "C" int vexb_bsr_create(int dev, void *stream, size_t nrows, size_t ncols, int block, const void *ptr, int ptr_bytes,
                               const void *col, int col_bytes, const void *val, int val_dtype, vexb_bspmat **out) {
    (void)stream;
    // every argument is checked before a device is touched (tests/test_bsr_oracle.py runs these checks without one)
    VEXB_CHECK(out, "out is NULL");
    *out = nullptr;
    VEXB_CHECK(block >= 2 && block <= 4, "block size %d is not 2, 3 or 4", block);
    VEXB_CHECK(val_dtype == VEXB_F64 || val_dtype == VEXB_F32, "values must be f64 or f32");
    sell_host h;
    VEXB_TRY(sell_check(nrows, ncols, ptr, ptr_bytes, col, col_bytes, val, "block ", h));

    DeviceGuard g(dev);
    if (!g.ok) VEXB_FAIL(VEXB_ERR_CUDA, "cannot select device %d", dev);
    vexb_bspmat *A = new vexb_bspmat;
    A->dev = dev; A->block = block; A->val_dtype = val_dtype;
    A->nrows = nrows; A->ncols = ncols; A->nnzb = h.nnz;
    const int st = sell_upload(A, h, val, dtype_size(val_dtype), (size_t)block * block);
    if (st != VEXB_OK) { vexb_bspmat_destroy(A); return st; }
    *out = A;
    return VEXB_OK;
}

extern "C" int vexb_bspmat_destroy(vexb_bspmat *A) {
    if (!A) return VEXB_OK;
    VEXB_RELEASE_GUARD();
    DeviceGuard g(A->dev);
    sell_free(A);
    delete A;
    return VEXB_OK;
}

extern "C" int vexb_bspmat_get_info(const vexb_bspmat *A, vexb_bspmat_info *info) {
    VEXB_CHECK(A && info, "NULL argument");
    memset(info, 0, sizeof(*info));
    info->nrows = A->nrows; info->ncols = A->ncols; info->nnzb = A->nnzb;
    info->block = A->block; info->val_dtype = A->val_dtype;
    info->n_slices = A->n_slices; info->n_slots = A->n_slots; info->device_bytes = A->device_bytes;
    return VEXB_OK;
}

extern "C" int vexb_bspmv(int dev, void *stream, const vexb_bspmat *A, const void *x, void *y, double alpha, int append) {
    VEXB_CHECK(A, "matrix is NULL");
    VEXB_CHECK(dev == A->dev, "matrix lives on device %d, not %d", A->dev, dev);
    VEXB_CHECK(A->nrows == 0 || y, "y is NULL");
    VEXB_CHECK(A->nnzb == 0 || x, "x is NULL");
    DeviceGuard g(dev); VEXB_CHECK(g.ok, "cannot select device %d", dev);
    if (A->val_dtype == VEXB_F64) return bspmv_launch<double>(A, (cudaStream_t)stream, (const double *)x, (double *)y, alpha, append);
    return bspmv_launch<float>(A, (cudaStream_t)stream, (const float *)x, (float *)y, (float)alpha, append);
}

extern "C" int vexb_zsr_create(int dev, void *stream, size_t nrows, size_t ncols, const void *ptr, int ptr_bytes,
                               const void *col, int col_bytes, const void *val, int val_dtype, vexb_zspmat **out) {
    (void)stream;
    // every argument is checked before a device is touched (tests/test_zsr_oracle.py runs these checks without one)
    VEXB_CHECK(out, "out is NULL");
    *out = nullptr;
    VEXB_CHECK(val_dtype == VEXB_F64 || val_dtype == VEXB_F32, "values must be f64 or f32");
    sell_host h;
    VEXB_TRY(sell_check(nrows, ncols, ptr, ptr_bytes, col, col_bytes, val, "", h));

    DeviceGuard g(dev);
    if (!g.ok) VEXB_FAIL(VEXB_ERR_CUDA, "cannot select device %d", dev);
    vexb_zspmat *A = new vexb_zspmat;
    A->dev = dev; A->val_dtype = val_dtype;
    A->nrows = nrows; A->ncols = ncols; A->nnz = h.nnz;
    const int st = sell_upload(A, h, val, dtype_size(val_dtype), 2);   // (re, im) of each entry: the bytes of std::complex<T>
    if (st != VEXB_OK) { vexb_zspmat_destroy(A); return st; }
    *out = A;
    return VEXB_OK;
}

extern "C" int vexb_zspmat_destroy(vexb_zspmat *A) {
    if (!A) return VEXB_OK;
    VEXB_RELEASE_GUARD();
    DeviceGuard g(A->dev);
    sell_free(A);
    delete A;
    return VEXB_OK;
}

extern "C" int vexb_zspmat_get_info(const vexb_zspmat *A, vexb_zspmat_info *info) {
    VEXB_CHECK(A && info, "NULL argument");
    memset(info, 0, sizeof(*info));
    info->nrows = A->nrows; info->ncols = A->ncols; info->nnz = A->nnz;
    info->val_dtype = A->val_dtype;
    info->n_slices = A->n_slices; info->n_slots = A->n_slots; info->device_bytes = A->device_bytes;
    return VEXB_OK;
}

extern "C" int vexb_zspmv(int dev, void *stream, const vexb_zspmat *A, const void *x, void *y, double alpha, int append) {
    VEXB_CHECK(A, "matrix is NULL");
    VEXB_CHECK(dev == A->dev, "matrix lives on device %d, not %d", A->dev, dev);
    VEXB_CHECK(A->nrows == 0 || y, "y is NULL");
    VEXB_CHECK(A->nnz == 0 || x, "x is NULL");
    const size_t pair = A->val_dtype == VEXB_F64 ? 2 * sizeof(double) : 2 * sizeof(float);
    VEXB_CHECK(A->nnz == 0 || (uintptr_t)x % pair == 0, "x is not aligned to one complex element (%zu bytes)", pair);
    DeviceGuard g(dev); VEXB_CHECK(g.ok, "cannot select device %d", dev);
    if (A->val_dtype == VEXB_F64) return zspmv_launch<double>(A, (cudaStream_t)stream, (const double *)x, (double *)y, alpha, append);
    return zspmv_launch<float>(A, (cudaStream_t)stream, (const float *)x, (float *)y, (float)alpha, append);
}

// ---- user value types -------------------------------------------------------------------------------------------------
namespace vexb {

// Slots in flight per loop turn of the generated kernel: U * (1 value + 1 column) streaming loads and U gathers of x per
// lane.  No spills for the 2 x 2 block (double4 / double2) or the complex (double2) type in either precision
// (-Xptxas -v on the generated source, DESIGN.md section 3 lists the register counts).
constexpr int kUsellUnroll = 4;

// Device type names are spelled by the user's type_name_impl: identifiers, possibly qualified or with spaces
// ("unsigned int").  Anything else (a brace, a semicolon) would put code outside the snippets.
static bool type_name_ok(const char *t) {
    if (!t || !*t) return false;
    for (const char *c = t; *c; ++c)
        if (!isalnum((unsigned char)*c) && *c != '_' && *c != ':' && *c != ' ') return false;
    return true;
}

static int usr_check_ops(const vexb_usr_ops *o) {
    VEXB_CHECK(o, "ops is NULL");
    VEXB_CHECK(type_name_ok(o->val_type), "val_type is not a type name");
    VEXB_CHECK(type_name_ok(o->rhs_type), "rhs_type is not a type name");
    VEXB_CHECK(o->rhs_bytes >= 1 && o->rhs_bytes <= 64, "rhs_bytes %zu is not in 1..64", o->rhs_bytes);
    VEXB_CHECK(o->decl && o->product && o->append, "a snippet of ops is NULL");
    return VEXB_OK;
}

// Alignment of a device vector type of `bytes` bytes (double2: 16, double3: 8, float2: 8, float3: 4, double4: 16).
static size_t natural_align(size_t bytes) {
    size_t a = 1;
    while (a < 16 && bytes % (2 * a) == 0) a *= 2;
    return a;
}

// The product kernel of a user strip (one warp per slice, one lane per row, as zsell_kernel), with the spmv_ops_impl
// snippets of the value type V and the vector type X, which use the names `sum` (accumulator), `v` (matrix value), `xv`
// (x at its column) and `t` (the old y_r in y += A x).  Per row, in storage order: decl; then for every stored value
// append_product(sum, v, xv); then y_r = sum, or t = y_r, append(t, sum), y_r = t.  Padding slots are skipped.
static std::string usr_source(const vexb_usr_ops &o, size_t val_bytes) {
    const int U = kUsellUnroll;
    std::ostringstream s;
    s << "// generated by libvexb200 (csrc/bspmv.cu): sliced-ELL product of a user value type\n"
         "typedef " << o.val_type << " vexb_val_t;\n"
         "typedef " << o.rhs_type << " vexb_rhs_t;\n"
         "static_assert(sizeof(vexb_val_t) == " << val_bytes << " && sizeof(vexb_rhs_t) == " << o.rhs_bytes << ",\n"
         "              \"the device types " << o.val_type << " and " << o.rhs_type << " must have the sizes of the host value "
         "(" << val_bytes << " bytes) and vector (" << o.rhs_bytes << " bytes) types\");\n"
         "extern \"C\" __global__ void __launch_bounds__(256) vexb_usr_kernel(unsigned long long n_slices_,\n"
         "    const int *__restrict__ slice_ptr_, const int *__restrict__ perm_, const int *__restrict__ col_,\n"
         "    const vexb_val_t *__restrict__ val_, const vexb_rhs_t *__restrict__ x_, vexb_rhs_t *y_, int append_) {\n"
         "  const unsigned long long s_ = (unsigned long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);\n"
         "  if (s_ >= n_slices_) return;\n"
         "  const int lane_ = threadIdx.x & 31;\n"
         "  const int base_ = __ldg(slice_ptr_ + s_), w_ = (__ldg(slice_ptr_ + s_ + 1) - base_) >> 5;\n"
         "  const int *cp_ = col_ + base_ + lane_;\n"
         "  const vexb_val_t *vp_ = val_ + (unsigned long long)base_ + lane_;\n" << o.decl << "\n"
         "  int k_ = 0;\n"
         "  for (; k_ + " << U << " <= w_; k_ += " << U << ") {\n"
         "    int c_[" << U << "]; vexb_val_t a_[" << U << "]; vexb_rhs_t b_[" << U << "];\n"
         "#pragma unroll\n"
         "    for (int u_ = 0; u_ < " << U << "; ++u_) { c_[u_] = __ldcs(cp_ + (k_ + u_) * 32); a_[u_] = vp_[(unsigned long long)(k_ + u_) * 32]; }\n"
         "#pragma unroll\n"
         "    for (int u_ = 0; u_ < " << U << "; ++u_) if (c_[u_] != -1) b_[u_] = x_[c_[u_]];\n"
         "#pragma unroll\n"
         "    for (int u_ = 0; u_ < " << U << "; ++u_) if (c_[u_] != -1) {\n"
         "      const vexb_val_t v = a_[u_]; const vexb_rhs_t xv = b_[u_];\n" << o.product << "\n"
         "    }\n"
         "  }\n"
         "  for (; k_ < w_; ++k_) {\n"
         "    const int c_ = __ldcs(cp_ + k_ * 32);\n"
         "    const vexb_val_t a_ = vp_[(unsigned long long)k_ * 32];\n"
         "    if (c_ != -1) {\n"
         "      const vexb_val_t v = a_; const vexb_rhs_t xv = x_[c_];\n" << o.product << "\n"
         "    }\n"
         "  }\n"
         "  const int r_ = __ldcs(perm_ + s_ * 32 + lane_);\n"     // read last: a register less through the loops
         "  if (r_ >= 0) {\n"
         "    if (append_) {\n"
         "      vexb_rhs_t t = y_[r_];\n" << o.append << "\n"
         "      y_[r_] = t;\n"
         "    } else {\n"
         "      y_[r_] = sum;\n"
         "    }\n"
         "  }\n"
         "}\n";
    return s.str();
}

// One kernel per (snippets, val_bytes): the front ends pass the same ops on every call.  The device's program header goes
// first in the source (the snippets may use what it declares).
static int usr_kernel(int dev, const vexb_usr_ops &o, size_t val_bytes, void **fn) {
    std::string key = "usr:";
    for (const char *part : {o.val_type, o.rhs_type, o.decl, o.product, o.append}) {
        key += std::to_string(strlen(part)); key += ':'; key += part;
    }
    key += std::to_string(o.rhs_bytes) + ":" + std::to_string(val_bytes);
    return jit_program(dev, key, "vexb_usr_kernel", program_header(dev), [&](JitBuild *b) {
        b->text = usr_source(o, val_bytes);
        return VEXB_OK;
    }, true, fn);
}

} // namespace vexb

extern "C" int vexb_usr_create(int dev, void *stream, size_t nrows, size_t ncols, const void *ptr, int ptr_bytes,
                               const void *col, int col_bytes, const void *val, int val_bytes, vexb_usrmat **out) {
    (void)stream;
    // every argument is checked before a device is touched (tests/test_usr_jit_cpu.py runs these checks without one)
    VEXB_CHECK(out, "out is NULL");
    *out = nullptr;
    VEXB_CHECK(val_bytes >= 1 && val_bytes <= 64 && val_bytes % 4 == 0, "val_bytes %d is not a multiple of 4 in 4..64", val_bytes);
    sell_host h;
    VEXB_TRY(sell_check(nrows, ncols, ptr, ptr_bytes, col, col_bytes, val, "", h));

    DeviceGuard g(dev);
    if (!g.ok) VEXB_FAIL(VEXB_ERR_CUDA, "cannot select device %d", dev);
    vexb_usrmat *A = new vexb_usrmat;
    A->dev = dev; A->val_bytes = val_bytes;
    A->nrows = nrows; A->ncols = ncols; A->nnz = h.nnz;
    const int st = sell_upload(A, h, val, (size_t)val_bytes, 1);
    if (st != VEXB_OK) { vexb_usrmat_destroy(A); return st; }
    *out = A;
    return VEXB_OK;
}

extern "C" int vexb_usrmat_destroy(vexb_usrmat *A) {
    if (!A) return VEXB_OK;
    VEXB_RELEASE_GUARD();
    DeviceGuard g(A->dev);
    sell_free(A);
    delete A;
    return VEXB_OK;
}

extern "C" int vexb_usrmat_get_info(const vexb_usrmat *A, vexb_usrmat_info *info) {
    VEXB_CHECK(A && info, "NULL argument");
    memset(info, 0, sizeof(*info));
    info->nrows = A->nrows; info->ncols = A->ncols; info->nnz = A->nnz;
    info->val_bytes = A->val_bytes;
    info->n_slices = A->n_slices; info->n_slots = A->n_slots; info->device_bytes = A->device_bytes;
    return VEXB_OK;
}

extern "C" int vexb_usr_spmv(int dev, void *stream, const vexb_usrmat *A, const vexb_usr_ops *ops, const void *x, void *y, int append) {
    VEXB_CHECK(A, "matrix is NULL");
    VEXB_TRY(usr_check_ops(ops));
    VEXB_CHECK(dev == A->dev, "matrix lives on device %d, not %d", A->dev, dev);
    VEXB_CHECK(A->nrows == 0 || y, "y is NULL");
    VEXB_CHECK(A->nnz == 0 || x, "x is NULL");
    const size_t al = natural_align(ops->rhs_bytes);
    VEXB_CHECK((uintptr_t)x % al == 0 && (uintptr_t)y % al == 0, "x and y must be aligned to %zu bytes", al);
    DeviceGuard g(dev); VEXB_CHECK(g.ok, "cannot select device %d", dev);
    if (A->nrows == 0) return VEXB_OK;
    cudaStream_t st = (cudaStream_t)stream;
    if (A->nnz == 0) {
        // as vexb_spmv on an empty strip: y = A*x zeroes y, y += A*x leaves it alone
        if (!append) VEXB_CUDA(cudaMemsetAsync(y, 0, A->nrows * ops->rhs_bytes, st));
        return VEXB_OK;
    }
    void *fn = nullptr;
    VEXB_TRY(usr_kernel(dev, *ops, (size_t)A->val_bytes, &fn));
    unsigned long long ns = A->n_slices;
    const void *sp = A->slice_ptr, *pm = A->perm, *cl = A->col, *vl = A->val;
    int ap = append ? 1 : 0;
    void *args[] = {&ns, &sp, &pm, &cl, &vl, &x, &y, &ap};
    return jit_launch(fn, (unsigned)((A->n_slices + 7) / 8), 256, 0, st, args);
}

extern "C" int vexb_jit_source_usr(const vexb_usr_ops *ops, int val_bytes, char *buf, size_t *len, int compile) {
    VEXB_CHECK(len, "len is NULL");
    VEXB_TRY(usr_check_ops(ops));
    VEXB_CHECK(val_bytes >= 1 && val_bytes <= 64 && val_bytes % 4 == 0, "val_bytes %d is not a multiple of 4 in 4..64", val_bytes);
    return jit_print(usr_source(*ops, (size_t)val_bytes), compile, false, buf, len);
}
