// Block sparse strips on one device: y (=|+=) alpha * A * x with B x B blocks (B = 2, 3, 4) as values, the product
// of vex::sparse::{csr, ell, matrix}<std::array<std::array<T,B>,B>> (the reference's custom value types,
// sparse/distributed.hpp:17-21 rhs_of + sparse/spmv_ops.hpp spmv_ops_impl).
//
// Layout: sliced ELL (SELL-32-sigma, as VEXB_FMT_SELL) over BLOCK rows, from the same host sell_layout, sigma
// ("spmv.sell_sigma") and perm / slice_ptr.  One int32 block column per slot (-1 = padding).  Values are planar per
// slot: component c = r*B + q of slot k, lane l of slice s sits at val[(slice_ptr[s] + 32k) * B*B + 32c + l], so every
// value load of a warp is 32 consecutive T whatever B is.  One column and one gather of B consecutive x values serve
// B*B values: 8B^2 + 4 bytes per stored block in double against 12B^2 for the same block expanded into scalar CSR.
#include "hostlogic.hpp"
#include "spmv_dev.cuh"
#include <vector>

struct vexb_bspmat {
    int dev = 0, block = 0, val_dtype = VEXB_F64;
    size_t nrows = 0, ncols = 0, nnzb = 0;     // block rows, block columns, stored blocks
    int *slice_ptr = nullptr, *perm = nullptr, *col = nullptr; void *val = nullptr;
    size_t n_slices = 0, n_slots = 0, device_bytes = 0;
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

template <class E>
static int upload_array(const std::vector<E> &h, void **d, size_t *bytes_acc) {
    *d = nullptr;
    if (h.empty()) return VEXB_OK;
    VEXB_CUDA(cudaMalloc(d, h.size() * sizeof(E)));
    VEXB_CUDA(cudaMemcpy(*d, h.data(), h.size() * sizeof(E), cudaMemcpyHostToDevice));
    *bytes_acc += h.size() * sizeof(E);
    return VEXB_OK;
}

// Host packing of the planar slots (see the top of this file); padding slots keep column -1 and zero values.
template <class T>
static int bsr_upload(vexb_bspmat *A, const std::vector<int> &rp, const std::vector<int> &bcol, const T *val,
                      const std::vector<int> &perm, const std::vector<int> &sptr) {
    const size_t B = (size_t)A->block, BB = B * B;
    std::vector<int> scol(A->n_slots, -1);
    std::vector<T> sval(A->n_slots * BB, T(0));
    for (size_t sl = 0; sl < A->n_slices; ++sl)
        for (int l = 0; l < 32; ++l) {
            const int r = perm[sl * 32 + l];
            if (r < 0) continue;
            for (int j = rp[r], k = 0; j < rp[r + 1]; ++j, ++k) {
                const size_t slot = (size_t)sptr[sl] + (size_t)k * 32;
                scol[slot + l] = bcol[j];
                for (size_t c = 0; c < BB; ++c) sval[slot * BB + 32 * c + l] = val[(size_t)j * BB + c];
            }
        }
    VEXB_TRY(upload_array(sptr, (void **)&A->slice_ptr, &A->device_bytes));
    VEXB_TRY(upload_array(perm, (void **)&A->perm, &A->device_bytes));
    VEXB_TRY(upload_array(scol, (void **)&A->col, &A->device_bytes));
    VEXB_TRY(upload_array(sval, &A->val, &A->device_bytes));
    return VEXB_OK;
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
    VEXB_CHECK(ptr_bytes == 4 || ptr_bytes == 8, "ptr_bytes must be 4 or 8");
    VEXB_CHECK(col_bytes == 4 || col_bytes == 8, "col_bytes must be 4 or 8");
    VEXB_CHECK(nrows == 0 || ptr, "ptr is NULL");
    VEXB_CHECK(nrows < (size_t)INT32_MAX && ncols < (size_t)INT32_MAX, "block dimensions exceed 32-bit local indices");
    const int64_t p0 = nrows ? read_index(ptr, ptr_bytes, 0) : 0;
    const int64_t nnzb = nrows ? read_index(ptr, ptr_bytes, nrows) - p0 : 0;
    VEXB_CHECK(nnzb >= 0 && nnzb < (int64_t)INT32_MAX - 64, "nnzb=%lld does not fit 32-bit row pointers", (long long)nnzb);
    VEXB_CHECK(nnzb == 0 || (col && val), "col/val is NULL");
    std::vector<int> rp(nrows + 1, 0), c((size_t)nnzb);
    for (size_t i = 1; i <= nrows; ++i) {
        const int64_t v = read_index(ptr, ptr_bytes, i) - p0;
        VEXB_CHECK(v >= rp[i - 1] && v <= nnzb, "row pointers decrease at block row %zu", i);
        rp[i] = (int)v;
    }
    for (size_t j = 0; j < (size_t)nnzb; ++j) {
        const int64_t cj = read_index(col, col_bytes, j);
        VEXB_CHECK(cj >= 0 && (size_t)cj < ncols, "block column %lld out of range at block %zu", (long long)cj, j);
        c[j] = (int)cj;
    }
    std::vector<int> perm, sptr;
    size_t slots = 0;
    VEXB_CHECK(sell_layout(nrows, rp.data(), param("spmv.sell_sigma", 1024), perm, sptr, &slots),
               "block strip too large for 32-bit slot offsets");

    DeviceGuard g(dev);
    if (!g.ok) VEXB_FAIL(VEXB_ERR_CUDA, "cannot select device %d", dev);
    vexb_bspmat *A = new vexb_bspmat;
    A->dev = dev; A->block = block; A->val_dtype = val_dtype;
    A->nrows = nrows; A->ncols = ncols; A->nnzb = (size_t)nnzb;
    A->n_slices = sptr.size() - 1; A->n_slots = slots;
    const int st = val_dtype == VEXB_F64 ? bsr_upload<double>(A, rp, c, (const double *)val, perm, sptr)
                                         : bsr_upload<float>(A, rp, c, (const float *)val, perm, sptr);
    if (st != VEXB_OK) { vexb_bspmat_destroy(A); return st; }
    *out = A;
    return VEXB_OK;
}

extern "C" int vexb_bspmat_destroy(vexb_bspmat *A) {
    if (!A) return VEXB_OK;
    VEXB_RELEASE_GUARD();
    DeviceGuard g(A->dev);
    cudaFree(A->slice_ptr); cudaFree(A->perm); cudaFree(A->col); cudaFree(A->val);
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
