// Device helpers shared by the sparse kernels (spmv.cu, distapply.cu): unfused arithmetic, L2 cache policies,
// streaming / keeping loads, the ELL row body.
#pragma once
#include "common.cuh"
#include "spmat.hpp"
#include <type_traits>

namespace vexb {

template <class T> __device__ __forceinline__ T t_mul(T a, T b);
template <> __device__ __forceinline__ double t_mul<double>(double a, double b) { return __dmul_rn(a, b); }
template <> __device__ __forceinline__ float t_mul<float>(float a, float b) { return __fmul_rn(a, b); }
template <class T> __device__ __forceinline__ T t_add(T a, T b);
template <> __device__ __forceinline__ double t_add<double>(double a, double b) { return __dadd_rn(a, b); }
template <> __device__ __forceinline__ float t_add<float>(float a, float b) { return __fadd_rn(a, b); }
template <class T> __device__ __forceinline__ T t_sub(T a, T b);
template <> __device__ __forceinline__ double t_sub<double>(double a, double b) { return __dsub_rn(a, b); }
template <> __device__ __forceinline__ float t_sub<float>(float a, float b) { return __fsub_rn(a, b); }

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

// L2 residency control.  The matrix streams through once per product, x is gathered ~nnz/ncols
// times: matrix traffic is marked evict-first and x evict-last, so the stream does not push x out
// of the 50 MB L2 (x gathers that miss L1 then cost an L2 hit, not an HBM round trip).
__device__ __forceinline__ uint64_t l2_policy_stream() {
    uint64_t p; asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p)); return p;
}
__device__ __forceinline__ uint64_t l2_policy_keep() {
    uint64_t p; asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p)); return p;
}

__device__ __forceinline__ void bulk_g2s(void *dst_smem, const void *src, uint32_t bytes, uint64_t *bar, uint64_t policy) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;"
                 :: "r"(smem_u32(dst_smem)), "l"(src), "r"(bytes), "r"(smem_u32(bar)), "l"(policy) : "memory");
}

// Asks L2 to fetch the 16-byte-aligned part of p[lo, hi), clipped to p[0, end).  A hint: no data comes back, no
// register waits for it, and nothing outside p[0, end) is touched.
template <class E>
__device__ __forceinline__ void prefetch_l2(const E *p, long long lo, long long hi, long long end, uint64_t policy) {
    lo = max(lo, 0ll); hi = min(hi, end);
    if (hi <= lo) return;
    const uintptr_t a = ((uintptr_t)(p + lo) + 15) & ~(uintptr_t)15, b = (uintptr_t)(p + hi) & ~(uintptr_t)15;
    if (b > a)
        asm volatile("cp.async.bulk.prefetch.L2.global.L2::cache_hint [%0], %1, %2;"
                     :: "l"(a), "r"((uint32_t)(b - a)), "l"(policy) : "memory");
}

__device__ __forceinline__ double ldg_keep(const double *p, uint64_t policy) {
    double v; asm volatile("ld.global.nc.L2::cache_hint.f64 %0, [%1], %2;" : "=d"(v) : "l"(p), "l"(policy)); return v;
}
__device__ __forceinline__ float ldg_keep(const float *p, uint64_t policy) {
    float v; asm volatile("ld.global.nc.L2::cache_hint.f32 %0, [%1], %2;" : "=f"(v) : "l"(p), "l"(policy)); return v;
}
// (re, im) of a complex element in one 16- or 8-byte load; p must be aligned to the pair
__device__ __forceinline__ double2 ldg_keep(const double2 *p, uint64_t policy) {
    double2 v; asm volatile("ld.global.nc.L2::cache_hint.v2.f64 {%0, %1}, [%2], %3;" : "=d"(v.x), "=d"(v.y) : "l"(p), "l"(policy)); return v;
}
__device__ __forceinline__ float2 ldg_keep(const float2 *p, uint64_t policy) {
    float2 v; asm volatile("ld.global.nc.L2::cache_hint.v2.f32 {%0, %1}, [%2], %3;" : "=f"(v.x), "=f"(v.y) : "l"(p), "l"(policy)); return v;
}
__device__ __forceinline__ int ldg_stream(const int *p, uint64_t policy) {
    int v; asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.s32 %0, [%1], %2;" : "=r"(v) : "l"(p), "l"(policy)); return v;
}
__device__ __forceinline__ short ldg_stream(const short *p, uint64_t policy) {
    short v; asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.s16 %0, [%1], %2;" : "=h"(v) : "l"(p), "l"(policy)); return v;
}
// Column of an ELL slot.  32-bit storage holds it directly (-1 = padding); 16-bit storage (spmv.col16) holds its
// distance from (row + shift of its slot), with -32768 = padding: 2 bytes less HBM traffic per stored entry for banded matrices.
__device__ __forceinline__ int ell_column(int raw, size_t, int) { return raw; }
__device__ __forceinline__ int ell_shift_of(const EllShifts &sh, int slot) { return sh.s[slot < kEllShiftSlots ? slot : kEllShiftSlots - 1]; }
__device__ __forceinline__ int ell_column(short raw, size_t row, int shift) { return raw == (short)-32768 ? -1 : (int)row + shift + (int)raw; }
__device__ __forceinline__ unsigned ldg_stream(const EllDiag *p, uint64_t policy) {
    unsigned v; asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.u8 %0, [%1], %2;" : "=r"(v) : "l"(p), "l"(policy)); return v;
}
// What a row reads once before its slots: the slot mask in the diagonal encoding (spmv.ell_diag), nothing otherwise.
__device__ __forceinline__ unsigned ell_row_mask(const int *, size_t, uint64_t) { return 0u; }
__device__ __forceinline__ unsigned ell_row_mask(const short *, size_t, uint64_t) { return 0u; }
__device__ __forceinline__ unsigned ell_row_mask(const EllDiag *m, size_t row, uint64_t policy) { return ldg_stream(m + row, policy); }
// Column of slot j of a row (-1 = padding) in each encoding.  The diagonal encoding reads no column stream: the entry of
// slot j, if its mask bit is set, sits at row + shift of slot j.
__device__ __forceinline__ int ell_slot_column(const int *col, size_t row, size_t pitch, int j, int, unsigned, uint64_t policy) {
    return ldg_stream(col + row + (size_t)j * pitch, policy);
}
__device__ __forceinline__ int ell_slot_column(const short *col, size_t row, size_t pitch, int j, int shift, unsigned, uint64_t policy) {
    return ell_column(ldg_stream(col + row + (size_t)j * pitch, policy), row, shift);
}
__device__ __forceinline__ int ell_slot_column(const EllDiag *, size_t row, size_t, int j, int shift, unsigned mask, uint64_t) {
    return (mask >> j) & 1u ? (int)row + shift : -1;
}
__device__ __forceinline__ double ldg_stream(const double *p, uint64_t policy) {
    double v; asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.f64 %0, [%1], %2;" : "=d"(v) : "l"(p), "l"(policy)); return v;
}
__device__ __forceinline__ float ldg_stream(const float *p, uint64_t policy) {
    float v; asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.f32 %0, [%1], %2;" : "=f"(v) : "l"(p), "l"(policy)); return v;
}
__device__ __forceinline__ unsigned ldg_stream(const EllClass *p, uint64_t policy) {
    unsigned v; asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.u8 %0, [%1], %2;" : "=r"(v) : "l"(p), "l"(policy)); return v;
}
// Class-table lookups (L1-resident, a broadcast when a warp's rows share a class).  volatile like the gathers of x, so
// the compiler keeps them after those: a lookup waits for the row's class byte, and the gathers must not wait with it.
__device__ __forceinline__ unsigned ldg_table(const unsigned char *p) {
    unsigned v; asm volatile("ld.global.nc.u8 %0, [%1];" : "=r"(v) : "l"(p)); return v;
}
__device__ __forceinline__ double ldg_table(const double *p) {
    double v; asm volatile("ld.global.nc.f64 %0, [%1];" : "=d"(v) : "l"(p)); return v;
}
__device__ __forceinline__ float ldg_table(const float *p) {
    float v; asm volatile("ld.global.nc.f32 %0, [%1];" : "=f"(v) : "l"(p)); return v;
}

// Column that slot j of a row-class strip gathers whether or not the row's slot holds an entry: row + shift of slot j,
// clamped to the strip's largest column x_max (a negative column wraps around to a large unsigned one), so that
// a padding slot still reads inside x.
__device__ __forceinline__ unsigned ell_class_column(size_t row, const EllShifts &sh, int j) {
    return min((unsigned)((int)row + sh.s[j]), (unsigned)sh.x_max);
}

// R rows of a row-class strip (spmv.ell_classes), sum[r] for row i[r].  All R class bytes and all R*W gathers of x are
// issued before the first table lookup: the column of slot k is row + shift of slot k whatever the row's mask says, so
// the gathers need not wait for the class byte.  A gather whose slot is padding reads x at a clamped address (ell_class_column)
// and is never added.  The set slots are added in slot order with the stored values, then
// the CSR tail: the same bits as the other encodings.
template <class T, int W, int R>
__device__ __forceinline__ void hell_class_rows(const size_t (&i)[R], const EllClass *__restrict__ cls, const EllShifts &sh,
                                                const T *__restrict__ table, const int *__restrict__ tail_ptr,
                                                const int *__restrict__ tail_col, const T *__restrict__ tail_val,
                                                const T *__restrict__ x, uint64_t stream, uint64_t keep, T (&sum)[R]) {
    static_assert(W > 0 && W <= (int)kEllDiagMaxWidth, "row classes hold one slot mask byte: unrolled widths up to 8 only");
    unsigned id[R]; T xv[R][W];
#pragma unroll
    for (int r = 0; r < R; ++r) id[r] = ldg_stream(cls + i[r], stream);
#pragma unroll
    for (int r = 0; r < R; ++r)
#pragma unroll
        for (int j = 0; j < W; ++j) xv[r][j] = ldg_keep(x + ell_class_column(i[r], sh, j), keep);
#pragma unroll
    for (int r = 0; r < R; ++r) {
        const unsigned m = ldg_table(reinterpret_cast<const unsigned char *>(table) + id[r]);
        const T *v = table + kEllClassHeader / sizeof(T) + id[r] * W;
        sum[r] = T(0);
#pragma unroll
        for (int j = 0; j < W; ++j) if ((m >> j) & 1u) sum[r] = t_add<T>(sum[r], t_mul<T>(ldg_table(v + j), xv[r][j]));
        if (tail_ptr)
            for (int j = tail_ptr[i[r]], e = tail_ptr[i[r] + 1]; j < e; ++j) sum[r] = t_add<T>(sum[r], t_mul<T>(tail_val[j], __ldg(x + tail_col[j])));
    }
}

template <class T>
__device__ __forceinline__ void store_y(T *y, size_t r, T sum, T alpha, int append) {
    const T v = t_mul<T>(alpha, sum);
    y[r] = append ? t_add<T>(y[r], v) : v;
}

// One row of a hybrid-ELL strip (hybrid_ell.inl:252-268): ELL slots in order, then the CSR tail; products and sums rounded
// separately.  W > 0: fully unrolled, all 2W streaming loads and then the W gathers of x in flight at once.  Row-class
// strips: hell_class_rows for one row.  V: stored value type -- T, or float under double vectors (VEXB_FMT_VALUES_F32),
// widened exactly to T before its product.
template <class T, int W, class C, class V = T>
__device__ __forceinline__ T hell_row_sum(size_t i, size_t pitch, int w_dyn, const C *__restrict__ ell_col, const EllShifts &shift,
                                          const V *__restrict__ ell_val, const int *__restrict__ tail_ptr,
                                          const int *__restrict__ tail_col, const V *__restrict__ tail_val,
                                          const T *__restrict__ x, uint64_t stream, uint64_t keep) {
    static_assert(W > 0 || !std::is_same<C, EllDiag>::value, "the diagonal encoding needs one shift per slot: unrolled widths only");
    if constexpr (std::is_same<C, EllClass>::value) {
        static_assert(std::is_same<T, V>::value, "row classes keep their table in the vector type");
        const size_t rows[1] = {i};
        T s[1];
        hell_class_rows<T, W, 1>(rows, ell_col, shift, ell_val, tail_ptr, tail_col, tail_val, x, stream, keep, s);
        return s[0];
    } else {
        T sum = T(0);
        const unsigned mask = ell_row_mask(ell_col, i, stream);
        if (W > 0) {
            int c[W > 0 ? W : 1]; V v[W > 0 ? W : 1]; T xv[W > 0 ? W : 1];
#pragma unroll
            for (int j = 0; j < W; ++j) { c[j] = ell_slot_column(ell_col, i, pitch, j, ell_shift_of(shift, j), mask, stream); v[j] = ldg_stream(ell_val + i + (size_t)j * pitch, stream); }
#pragma unroll
            for (int j = 0; j < W; ++j) xv[j] = (c[j] != -1) ? ldg_keep(x + c[j], keep) : T(0);
#pragma unroll
            for (int j = 0; j < W; ++j) if (c[j] != -1) sum = t_add<T>(sum, t_mul<T>(T(v[j]), xv[j]));
        } else {
            // any width: plain dependent loop rather than batches of 4 columns: occupancy hides the latency, and a
            // padded slot (column -1) costs 4 bytes, not 12, because its value is never fetched.
            for (int j = 0; j < w_dyn; ++j) {
                const int c = ell_slot_column(ell_col, i, pitch, j, shift.s[0], mask, stream);   // run-time widths use one shift (spmv.cu build())
                if (c != -1) sum = t_add<T>(sum, t_mul<T>(T(ldg_stream(ell_val + i + (size_t)j * pitch, stream)), ldg_keep(x + c, keep)));
            }
        }
        if (tail_ptr) {
            for (int j = tail_ptr[i], e = tail_ptr[i + 1]; j < e; ++j) sum = t_add<T>(sum, t_mul<T>(T(tail_val[j]), __ldg(x + tail_col[j])));
        }
        return sum;
    }
}

} // namespace vexb
