// vex::SpMatCCSR (vexcl/spmat/ccsr.hpp:54-86; kernel text :176-201): "compressed CSR" for stencil-like matrices.
// Only the UNIQUE rows are stored, with column positions relative to the diagonal; idx[i] names the unique row of
// matrix row i:
//     y[i] = sum_{j in row[idx[i]] .. row[idx[i]+1]}  val[j] * x[i + col[j]]
//
// Design.  The product is HBM-bound on three streams: idx (read once), x (each element is needed by every row
// whose stencil touches it, served by L1/L2 after its first read) and y.  So
//   * idx is re-encoded at upload in the narrowest type that holds m unique rows (1 byte for m <= 256, which covers
//     every stencil): 17 B/row of compulsory traffic for double instead of 24 B with the reference's size_t idx;
//   * the unique-row table (a few dozen entries) is staged into shared memory once per block, so the inner loop is
//     one shared-memory broadcast and one cached global load per non-zero;
//   * one thread per row, consecutive threads on consecutive rows: every x access of a warp is one or two lines.
// Products and sums are rounded separately and accumulated in storage order (no FMA), so the result is
// bit-identical to the reference's loop compiled without contraction (oracle/ccsr.py).
#include <algorithm>
#include <mutex>
#include <string>
#include <vector>
#include "common.cuh"
#include "jit.hpp"
#include "ccsr.hpp"

struct vexb_ccsr {
    int dev = 0, val_dtype = VEXB_F64, idx_bytes = 1;
    size_t n = 0, m = 0, nnz = 0, device_bytes = 0;
    void *idx = nullptr; int *row = nullptr; int *col = nullptr; void *val = nullptr;
    bool table_in_smem = true;
    std::vector<int> hrow, hcol; std::vector<double> hval;    // host copy of the unique-row table (source of the specialised kernel)
    void *jit_fn = nullptr; bool jit_failed = false;
    void *term_desc = nullptr;                                 // {idx, row, col, val} in device memory, for VEXB_TERM_CCSR
};

namespace vexb {
namespace {

template <class T> __device__ __forceinline__ T c_mul(T a, T b);
template <> __device__ __forceinline__ double c_mul<double>(double a, double b) { return __dmul_rn(a, b); }
template <> __device__ __forceinline__ float c_mul<float>(float a, float b) { return __fmul_rn(a, b); }
template <class T> __device__ __forceinline__ T c_add(T a, T b);
template <> __device__ __forceinline__ double c_add<double>(double a, double b) { return __dadd_rn(a, b); }
template <> __device__ __forceinline__ float c_add<float>(float a, float b) { return __fadd_rn(a, b); }

constexpr size_t CCSR_SMEM_LIMIT = 40 * 1024;
constexpr long CCSR_DEFAULT_KERNEL = 1;
constexpr long CCSR_DEFAULT_JIT = 1;        // the matrix-specialised NVRTC kernel (same bits; the table kernel serves when NVRTC is missing or the table is large)

template <class T, class I, bool SMEM, int CCSR_THREADS, int CCSR_BATCH, bool HOIST>
__global__ void __launch_bounds__(CCSR_THREADS) ccsr_kernel(size_t n, int m, int nnz, const I *__restrict__ idx,
                                                            const int *__restrict__ row, const int *__restrict__ col,
                                                            const T *__restrict__ val, const T *__restrict__ x, T *y,
                                                            T alpha, int append) {
    extern __shared__ __align__(16) unsigned char smem[];
    const T *vs = val; const int *cs = col, *rs = row;
    const size_t i = (size_t)blockIdx.x * CCSR_THREADS + threadIdx.x;
    // HOIST: the two loads that depend on nothing (idx[i], and y[i] when appending) are issued before the table is
    // staged, so that a block waits for one DRAM round trip + the gathers instead of table -> idx -> gathers -> y.
    int u = 0; T yo = T(0);
    if (HOIST && i < n) { u = (int)idx[i]; if (append) yo = y[i]; }
    if (SMEM) {
        T *v = reinterpret_cast<T *>(smem);
        int *c = reinterpret_cast<int *>(v + nnz);
        int *r = c + nnz;
#pragma unroll 1
        for (int j = threadIdx.x; j < nnz; j += CCSR_THREADS) { v[j] = val[j]; c[j] = col[j]; }
#pragma unroll 1
        for (int j = threadIdx.x; j <= m; j += CCSR_THREADS) r[j] = row[j];
        __syncthreads();
        vs = v; cs = c; rs = r;
    }
    if (i >= n) return;
    if (!HOIST) u = (int)idx[i];
    T sum = T(0);
    // gathers of up to CCSR_BATCH entries are issued together (one dependent load per thread would leave the kernel
    // latency-bound); products are then accumulated
    // in storage order
    const T *xi = x + (ptrdiff_t)i;
    for (int j = rs[u], e = rs[u + 1]; j < e; j += CCSR_BATCH) {
        T xv[CCSR_BATCH];
#pragma unroll
        for (int k = 0; k < CCSR_BATCH; ++k) xv[k] = (j + k < e) ? __ldg(xi + cs[j + k]) : T(0);
#pragma unroll
        for (int k = 0; k < CCSR_BATCH; ++k) if (j + k < e) sum = c_add<T>(sum, c_mul<T>(vs[j + k], xv[k]));
    }
    const T v = c_mul<T>(alpha, sum);
    if (HOIST) y[i] = append ? c_add<T>(yo, v) : v;
    else y[i] = append ? c_add<T>(y[i], v) : v;
}

// Variant 2/3 (ccsr.kernel = 2 | 3).  Variant 1 is latency-bound -- each block walks a chain of four dependent memory
// latencies (table -> barrier -> idx -> x gathers -> y read-modify-write).  Here the idx and y loads
// are issued before the table is staged (chain of two), a table entry is one 16-byte shared-memory word {val, col}
// instead of two loads, and with ROWS = 2 every thread carries two rows so that the staging is paid half as often.
template <class T> struct Entry;
template <> struct __align__(16) Entry<double> { double v; int c; int pad; };
template <> struct __align__(8) Entry<float> { float v; int c; };

template <class T, class I, int THREADS, int ROWS>
__global__ void __launch_bounds__(THREADS) ccsr_kernel2(size_t n, int m, int nnz, const I *__restrict__ idx,
                                                        const int *__restrict__ row, const int *__restrict__ col,
                                                        const T *__restrict__ val, const T *__restrict__ x, T *y,
                                                        T alpha, int append) {
    extern __shared__ __align__(16) unsigned char smem[];
    Entry<T> *tab = reinterpret_cast<Entry<T> *>(smem);
    int *rs = reinterpret_cast<int *>(tab + nnz);
    const size_t base = (size_t)blockIdx.x * (THREADS * ROWS) + threadIdx.x;
    int u[ROWS]; T yo[ROWS];
#pragma unroll
    for (int r = 0; r < ROWS; ++r) {
        const size_t i = base + (size_t)r * THREADS;
        const bool ok = i < n;
        u[r] = ok ? (int)idx[i] : -1;
        yo[r] = (ok && append) ? y[i] : T(0);
    }
    for (int j = threadIdx.x; j < nnz; j += THREADS) { Entry<T> e; e.v = val[j]; e.c = col[j]; tab[j] = e; }
    for (int j = threadIdx.x; j <= m; j += THREADS) rs[j] = row[j];
    __syncthreads();
#pragma unroll
    for (int r = 0; r < ROWS; ++r) {
        if (u[r] < 0) continue;
        const size_t i = base + (size_t)r * THREADS;
        const T *xi = x + (ptrdiff_t)i;
        T sum = T(0);
        for (int j = rs[u[r]], e = rs[u[r] + 1]; j < e; j += 8) {
            Entry<T> t[8]; T xv[8];
#pragma unroll
            for (int k = 0; k < 8; ++k) if (j + k < e) { t[k] = tab[j + k]; xv[k] = __ldg(xi + t[k].c); }
#pragma unroll
            for (int k = 0; k < 8; ++k) if (j + k < e) sum = c_add<T>(sum, c_mul<T>(t[k].v, xv[k]));
        }
        const T v = c_mul<T>(alpha, sum);
        y[i] = append ? c_add<T>(yo[r], v) : v;
    }
}

template <class H> static int upload(const std::vector<H> &h, void **d, size_t *acc) {
    const size_t bytes = (h.size() ? h.size() : 1) * sizeof(H);
    VEXB_CUDA(cudaMalloc(d, bytes));
    if (!h.empty()) VEXB_CUDA(cudaMemcpy(*d, h.data(), h.size() * sizeof(H), cudaMemcpyHostToDevice));
    *acc += bytes;
    return VEXB_OK;
}

static long long read_int(const void *p, int bytes, bool is_signed, size_t k) {
    if (bytes == 4) return is_signed ? (long long)((const int32_t *)p)[k] : (long long)((const uint32_t *)p)[k];
    return is_signed ? (long long)((const int64_t *)p)[k] : (long long)((const uint64_t *)p)[k];
}

template <class T, class I, int THREADS, int BATCH, bool HOIST>
static int launch_cfg(const vexb_ccsr *A, cudaStream_t st, const T *x, T *y, T alpha, int append) {
    const unsigned blocks = (unsigned)((A->n + THREADS - 1) / THREADS);
    if (A->table_in_smem && param("ccsr.smem", 1)) {
        const size_t smem = A->nnz * (sizeof(T) + sizeof(int)) + (A->m + 1) * sizeof(int);
        ccsr_kernel<T, I, true, THREADS, BATCH, HOIST><<<blocks, THREADS, smem, st>>>(A->n, (int)A->m, (int)A->nnz, (const I *)A->idx, A->row, A->col,
                                                                             (const T *)A->val, x, y, alpha, append);
    } else {
        ccsr_kernel<T, I, false, THREADS, BATCH, HOIST><<<blocks, THREADS, 0, st>>>(A->n, (int)A->m, (int)A->nnz, (const I *)A->idx, A->row, A->col,
                                                                           (const T *)A->val, x, y, alpha, append);
    }
    VEXB_LAUNCHED();
    return VEXB_OK;
}

template <class T, class I, int ROWS>
static int launch2(const vexb_ccsr *A, cudaStream_t st, const T *x, T *y, T alpha, int append) {
    constexpr int THREADS = 256;
    const unsigned blocks = (unsigned)((A->n + THREADS * ROWS - 1) / (THREADS * ROWS));
    const size_t smem = A->nnz * sizeof(Entry<T>) + (A->m + 1) * sizeof(int);
    ccsr_kernel2<T, I, THREADS, ROWS><<<blocks, THREADS, smem, st>>>(A->n, (int)A->m, (int)A->nnz, (const I *)A->idx, A->row, A->col,
                                                                   (const T *)A->val, x, y, alpha, append);
    VEXB_LAUNCHED();
    return VEXB_OK;
}

template <class T, class I>
static int launch(const vexb_ccsr *A, cudaStream_t st, const T *x, T *y, T alpha, int append) {
    // tunables (vexb_set_param): ccsr.kernel = 1 | 2 | 3; for kernel 1: ccsr.threads = 256 | 1024, ccsr.batch = 8 | 1, ccsr.hoist = 1 | 0, ccsr.smem = 1 | 0
    long kernel = param("ccsr.kernel", 0);
    if (kernel <= 0) kernel = CCSR_DEFAULT_KERNEL;
    if (kernel >= 2 && A->nnz * sizeof(Entry<T>) + (A->m + 1) * sizeof(int) <= CCSR_SMEM_LIMIT)
        return kernel == 3 ? launch2<T, I, 2>(A, st, x, y, alpha, append) : launch2<T, I, 1>(A, st, x, y, alpha, append);
    const long threads = param("ccsr.threads", 256), batch = param("ccsr.batch", 8), hoist = param("ccsr.hoist", 1);
    if (threads == 1024) return launch_cfg<T, I, 1024, 8, true>(A, st, x, y, alpha, append);
    if (!hoist) return batch == 1 ? launch_cfg<T, I, 256, 1, false>(A, st, x, y, alpha, append) : launch_cfg<T, I, 256, 8, false>(A, st, x, y, alpha, append);
    return batch == 1 ? launch_cfg<T, I, 256, 1, true>(A, st, x, y, alpha, append) : launch_cfg<T, I, 256, 8, true>(A, st, x, y, alpha, append);
}

// ---- matrix-specialised kernel (ccsr.jit = 1; NVRTC) ----------------------------------------------------------------------
// The reference generates its CCSR product as source text per expression (ccsr.hpp:176-201) but still walks the row
// table at run time.  Here the unique rows themselves become code: one `case` per unique row with the column offsets
// as address immediates and the values as hexadecimal floating literals -- no table, no loop, no shared memory, about
// 25 instructions per row instead of ~190.  Same operation order and rounding as ccsr_kernel (products and sums
// separate, storage order), so the bits are identical.  Eligible when the table is small (CCSR_JIT_MAX_*).
constexpr size_t CCSR_JIT_MAX_ROWS = 32, CCSR_JIT_MAX_NNZ = 256;

// Rows per thread of the generated kernel: the product is two dependent memory round trips per row (idx[i], then the
// gathers); at one row per thread the kernel is bound by exactly that latency.  With R rows per thread the R idx bytes travel together, and when the R rows share a
// unique row (the rule on structured grids) all R * width gathers are in flight at once.
static int ccsr_jit_rows_per_thread(const std::vector<int> &row) {
    int maxw = 0;
    for (size_t u = 0; u + 1 < row.size(); ++u) maxw = std::max(maxw, row[u + 1] - row[u]);
    return maxw <= 8 ? 4 : maxw <= 16 ? 2 : 1;
}

static std::string ccsr_jit_source(int val_dtype, int idx_bytes, const std::vector<int> &row, const std::vector<int> &col,
                                   const std::vector<double> &val) {
    const bool f64 = val_dtype == VEXB_F64;
    const char *T = f64 ? "double" : "float";
    const char *I = idx_bytes == 1 ? "unsigned char" : idx_bytes == 2 ? "unsigned short" : "int";
    const char *mul = f64 ? "__dmul_rn" : "__fmul_rn", *add = f64 ? "__dadd_rn" : "__fadd_rn";
    const int R = ccsr_jit_rows_per_thread(row);
    const int minblocks = R == 4 ? 3 : R == 2 ? 4 : 8;
    std::string s;
    char buf[512];
    auto lit = [&](double v) { if (f64) snprintf(buf, sizeof(buf), "%a", v); else snprintf(buf, sizeof(buf), "%af", (double)(float)v); return std::string(buf); };
    // products of unique row u for the row whose variables carry the suffix k: gathers in groups of 8, then the products in order
    auto row_body = [&](size_t u, int k, const char *indent) {
        std::string r;
        for (int base = row[u]; base < row[u + 1]; base += 8) {
            const int end = std::min(base + 8, row[u + 1]);
            for (int j = base; j < end; ++j) {
                snprintf(buf, sizeof(buf), "%sconst %s x%d_%d = __ldg(xi%d + (%d));\n", indent, T, k, j - row[u], k, col[j]);
                r += buf;
            }
            for (int j = base; j < end; ++j) {
                const std::string v = lit(val[j]);
                snprintf(buf, sizeof(buf), "%ssum%d = %s(sum%d, %s(%s, x%d_%d));\n", indent, k, add, k, mul, v.c_str(), k, j - row[u]);
                r += buf;
            }
        }
        return r;
    };
    s += "// generated by libvexb200 (csrc/ccsr.cu) for one CCSR matrix: " + std::to_string(row.size() - 1) + " unique rows, " +
         std::to_string(col.size()) + " entries, " + std::to_string(R) + " rows per thread\n";
    snprintf(buf, sizeof(buf), "extern \"C\" __global__ void __launch_bounds__(256, %d) vexb_ccsr_jit(unsigned long long n, const %s *__restrict__ idx,\n"
                               "        const %s *__restrict__ x, %s *y, %s alpha, int append) {\n", minblocks, I, T, T, T);
    s += buf;
    snprintf(buf, sizeof(buf), "    const unsigned long long ib = (unsigned long long)blockIdx.x * %dull + threadIdx.x;\n    if (ib >= n) return;\n", 256 * R);
    s += buf;
    for (int k = 0; k < R; ++k) {
        snprintf(buf, sizeof(buf), "    const unsigned long long i%d = ib + %dull; const bool in%d = i%d < n;\n", k, 256 * k, k, k);
        s += buf;
    }
    for (int k = 0; k < R; ++k) { snprintf(buf, sizeof(buf), "    const int u%d = in%d ? (int)idx[i%d] : -1;\n", k, k, k); s += buf; }
    for (int k = 0; k < R; ++k) { snprintf(buf, sizeof(buf), "    %s yo%d = 0; if (append && in%d) yo%d = y[i%d];\n", T, k, k, k, k); s += buf; }
    for (int k = 0; k < R; ++k) { snprintf(buf, sizeof(buf), "    const %s *xi%d = x + i%d; %s sum%d = 0;\n", T, k, k, T, k); s += buf; }
    if (R > 1) {
        // fast path: the thread's rows share one unique row -> straight-line code, every gather issued before the first product
        s += "    if (";
        for (int k = 1; k < R; ++k) { snprintf(buf, sizeof(buf), "%su0 == u%d", k > 1 ? " && " : "", k); s += buf; }
        s += ") {\n        switch (u0) {\n";
        for (size_t u = 0; u + 1 < row.size(); ++u) {
            s += "        case " + std::to_string(u) + ": {\n";
            const int w = row[u + 1] - row[u];
            if (w <= 8) {
                // all R * w gathers, then the products row by row (each row's sum in storage order)
                for (int k = 0; k < R; ++k)
                    for (int j = row[u]; j < row[u + 1]; ++j) {
                        snprintf(buf, sizeof(buf), "            const %s x%d_%d = __ldg(xi%d + (%d));\n", T, k, j - row[u], k, col[j]);
                        s += buf;
                    }
                for (int k = 0; k < R; ++k)
                    for (int j = row[u]; j < row[u + 1]; ++j) {
                        const std::string v = lit(val[j]);
                        snprintf(buf, sizeof(buf), "            sum%d = %s(sum%d, %s(%s, x%d_%d));\n", k, add, k, mul, v.c_str(), k, j - row[u]);
                        s += buf;
                    }
            } else {
                for (int k = 0; k < R; ++k) s += row_body(u, k, "            ");
            }
            s += "        } break;\n";
        }
        s += "        default: break;\n        }\n    } else {\n";
    }
    for (int k = 0; k < R; ++k) {
        snprintf(buf, sizeof(buf), "        switch (u%d) {\n", k);
        s += buf;
        for (size_t u = 0; u + 1 < row.size(); ++u) {
            s += "        case " + std::to_string(u) + ": {\n" + row_body(u, k, "            ") + "        } break;\n";
        }
        s += "        default: break;\n        }\n";
    }
    if (R > 1) s += "    }\n";
    for (int k = 0; k < R; ++k) {
        snprintf(buf, sizeof(buf), "    if (in%d) { const %s v = %s(alpha, sum%d); y[i%d] = append ? %s(yo%d, v) : v; }\n", k, T, mul, k, k, add, k);
        s += buf;
    }
    s += "}\n";
    return s;
}

template <class T>
static int launch_jit(vexb_ccsr *A, cudaStream_t st, const T *x, T *y, T alpha, int append, bool *done) {
    *done = false;
    if (A->jit_failed || A->m > CCSR_JIT_MAX_ROWS || A->nnz > CCSR_JIT_MAX_NNZ) return VEXB_OK;
    if (!A->jit_fn) {
        const std::string src = ccsr_jit_source(A->val_dtype, A->idx_bytes, A->hrow, A->hcol, A->hval);
        if (jit_program(A->dev, "ccsr:" + src, "vexb_ccsr_jit", std::string(), [&](JitBuild *b) { b->text = src; return VEXB_OK; }, true,
                        &A->jit_fn) != VEXB_OK) { A->jit_failed = true; return VEXB_OK; }   // generic kernel instead
    }
    unsigned long long n = A->n;
    const void *idx = A->idx;
    void *args[] = {&n, &idx, &x, &y, &alpha, &append};
    const size_t per_block = 256 * (size_t)ccsr_jit_rows_per_thread(A->hrow);
    VEXB_TRY(jit_launch(A->jit_fn, (unsigned)((A->n + per_block - 1) / per_block), 256, 0, st, args));
    *done = true;
    return VEXB_OK;
}

template <class T>
static int launch_idx(const vexb_ccsr *A, cudaStream_t st, const T *x, T *y, T alpha, int append) {
    switch (A->idx_bytes) {
        case 1: return launch<T, uint8_t>(A, st, x, y, alpha, append);
        case 2: return launch<T, uint16_t>(A, st, x, y, alpha, append);
        default: return launch<T, int32_t>(A, st, x, y, alpha, append);
    }
}

} // namespace
} // namespace vexb

using namespace vexb;

extern "C" int vexb_ccsr_create(int dev, void *stream, size_t n, size_t m, const void *idx, int idx_bytes,
                                const void *row, int row_bytes, const void *col, int col_bytes,
                                const void *val, int val_dtype, vexb_ccsr **out) {
    (void)stream;
    return vexb::ccsr_create_ex(dev, n, n, m, idx, idx_bytes, row, row_bytes, col, col_bytes, val, val_dtype, out);
}

// n rows applied to a vector of xlen elements (xlen = n for vex::SpMatCCSR; a row strip of vex::SpMat stored as row
// patterns, spmv.cu, has xlen = the strip's local column count).
int vexb::ccsr_create_ex(int dev, size_t n, size_t xlen, size_t m, const void *idx, int idx_bytes,
                         const void *row, int row_bytes, const void *col, int col_bytes,
                         const void *val, int val_dtype, vexb_ccsr **out) {
    VEXB_CHECK(out, "null output handle");
    VEXB_CHECK((idx || !n) && row && (idx_bytes == 4 || idx_bytes == 8) && (row_bytes == 4 || row_bytes == 8) && (col_bytes == 4 || col_bytes == 8),
               "idx/row/col must be 32- or 64-bit integer arrays");
    VEXB_CHECK(val_dtype == VEXB_F64 || val_dtype == VEXB_F32, "CCSR values must be float or double");
    VEXB_CHECK(m >= 1 && m < (size_t)1 << 31 && n < (size_t)1 << 40, "CCSR dimensions out of range");
    const long long nnz = read_int(row, row_bytes, false, m);
    VEXB_CHECK(nnz >= 0 && nnz < (1LL << 31) && (col || !nnz) && (val || !nnz), "CCSR unique rows hold too many entries");
    std::vector<int> hrow(m + 1), hcol((size_t)nnz);
    for (size_t k = 0; k <= m; ++k) {
        const long long r = read_int(row, row_bytes, false, k);
        VEXB_CHECK(r >= 0 && r <= nnz && (k == 0 || r >= hrow[k - 1]), "CCSR row pointers must be non-decreasing");
        hrow[k] = (int)r;
    }
    VEXB_CHECK(hrow[0] == 0, "CCSR row pointers must start at 0");
    // reach of every unique row relative to the diagonal, from its own entries only (an empty row reaches nothing; a row
    // whose entries all lie left of the diagonal is fine for i >= xlen as long as i + hi stays inside x)
    std::vector<long long> lo(m, 0), hi(m, 0);
    for (size_t u = 0; u < m; ++u)
        for (int j = hrow[u]; j < hrow[u + 1]; ++j) {
            const long long c = read_int(col, col_bytes, true, (size_t)j);
            VEXB_CHECK(c > -(1LL << 31) && c < (1LL << 31), "CCSR column offset does not fit 32 bits");
            hcol[(size_t)j] = (int)c;
            if (j == hrow[u]) lo[u] = hi[u] = c;
            else { lo[u] = c < lo[u] ? c : lo[u]; hi[u] = c > hi[u] ? c : hi[u]; }
        }
    auto *A = new vexb_ccsr();
    A->dev = dev; A->val_dtype = val_dtype; A->n = n; A->m = m; A->nnz = (size_t)nnz;
    A->hrow = hrow; A->hcol = hcol; A->hval.resize((size_t)nnz);
    for (long long j = 0; j < nnz; ++j) A->hval[(size_t)j] = val_dtype == VEXB_F64 ? ((const double *)val)[j] : (double)((const float *)val)[j];
    A->idx_bytes = m <= 256 ? 1 : m <= 65536 ? 2 : 4;
    A->table_in_smem = A->nnz * (dtype_size(val_dtype) + sizeof(int)) + (m + 1) * sizeof(int) <= CCSR_SMEM_LIMIT;
    std::vector<uint8_t> i8; std::vector<uint16_t> i16; std::vector<int32_t> i32;
    if (A->idx_bytes == 1) i8.resize(n); else if (A->idx_bytes == 2) i16.resize(n); else i32.resize(n);
    for (size_t i = 0; i < n; ++i) {
        const long long u = read_int(idx, idx_bytes, false, i);
        if (!(u >= 0 && (size_t)u < m)) { delete A; VEXB_FAIL(VEXB_ERR_INVALID, "CCSR idx[%zu] = %lld names no unique row (m = %zu)", i, u, m); }
        // the reference reads x[i + col[j]] unchecked (ccsr.hpp:195); a matrix that reaches outside x is rejected here
        if (hrow[(size_t)u + 1] > hrow[(size_t)u] && ((long long)i + lo[(size_t)u] < 0 || (long long)i + hi[(size_t)u] >= (long long)xlen)) {
            delete A; VEXB_FAIL(VEXB_ERR_INVALID, "CCSR row %zu (unique row %lld) reaches outside the vector", i, u);
        }
        if (A->idx_bytes == 1) i8[i] = (uint8_t)u; else if (A->idx_bytes == 2) i16[i] = (uint16_t)u; else i32[i] = (int32_t)u;
    }
    DeviceGuard g(dev);
    if (!g.ok) { delete A; VEXB_FAIL(VEXB_ERR_INVALID, "cannot select device %d", dev); }
    int st = A->idx_bytes == 1 ? upload(i8, &A->idx, &A->device_bytes) : A->idx_bytes == 2 ? upload(i16, &A->idx, &A->device_bytes)
                                                                                          : upload(i32, &A->idx, &A->device_bytes);
    if (st == VEXB_OK) st = upload(hrow, (void **)&A->row, &A->device_bytes);
    if (st == VEXB_OK) st = upload(hcol, (void **)&A->col, &A->device_bytes);
    if (st == VEXB_OK) {
        if (val_dtype == VEXB_F64) { std::vector<double> v((const double *)val, (const double *)val + nnz); st = upload(v, &A->val, &A->device_bytes); }
        else { std::vector<float> v((const float *)val, (const float *)val + nnz); st = upload(v, &A->val, &A->device_bytes); }
    }
    if (st != VEXB_OK) { vexb_ccsr_destroy(A); return st; }
    *out = A;
    return VEXB_OK;
}

extern "C" int vexb_ccsr_destroy(vexb_ccsr *A) {
    if (!A) return VEXB_OK;
    VEXB_RELEASE_GUARD();
    DeviceGuard g(A->dev);
    cudaFree(A->idx); cudaFree(A->row); cudaFree(A->col); cudaFree(A->val); cudaFree(A->term_desc);
    delete A;
    return VEXB_OK;
}

int vexb::ccsr_term_check(const vexb_ccsr *A, int k, int dev, int dtype, int idx_bytes, size_t n, size_t index_offset) {
    VEXB_CHECK(A->dev == dev, "term %d: the CCSR matrix lives on device %d, not %d", k, A->dev, dev);
    VEXB_CHECK(A->val_dtype == dtype, "term %d: the CCSR matrix holds values of type %d, the terminal says %d", k, A->val_dtype, dtype);
    VEXB_CHECK(idx_bytes == A->idx_bytes, "term %d: the CCSR matrix stores idx in %d bytes, the terminal says %d", k, A->idx_bytes, idx_bytes);
    VEXB_CHECK(index_offset == 0 && n == A->n, "term %d: a CCSR product covers the whole matrix (%zu rows), not elements [%zu, %zu)",
               k, A->n, index_offset, index_offset + n);
    return VEXB_OK;
}

int vexb::ccsr_term_desc(const vexb_ccsr *A, void **desc) {
    static std::mutex mx;
    std::lock_guard<std::mutex> lock(mx);
    vexb_ccsr *M = const_cast<vexb_ccsr *>(A);                       // lazily attaches the descriptor
    if (!M->term_desc) {
        const void *h[4] = {A->idx, A->row, A->col, A->val};
        DeviceGuard g(A->dev); VEXB_CHECK(g.ok, "cannot select device %d", A->dev);
        void *d = nullptr;
        VEXB_CUDA(cudaMalloc(&d, sizeof(h)));
        const cudaError_t e = cudaMemcpy(d, h, sizeof(h), cudaMemcpyHostToDevice);
        if (e != cudaSuccess) { cudaFree(d); VEXB_FAIL(VEXB_ERR_CUDA, "CCSR terminal descriptor: %s", cudaGetErrorString(e)); }
        M->term_desc = d;
    }
    *desc = M->term_desc;
    return VEXB_OK;
}

extern "C" int vexb_ccsr_get_info(const vexb_ccsr *A, vexb_ccsr_info *info) {
    VEXB_CHECK(A && info, "null argument");
    info->nrows = A->n; info->unique_rows = A->m; info->nnz = A->nnz; info->idx_bytes = A->idx_bytes;
    info->table_in_smem = A->table_in_smem ? 1 : 0; info->device_bytes = A->device_bytes;
    return VEXB_OK;
}

extern "C" int vexb_ccsr_spmv(int dev, void *stream, const vexb_ccsr *A, const void *x, void *y, double alpha, int append) {
    VEXB_CHECK(A, "null matrix");
    VEXB_CHECK(dev == A->dev, "matrix lives on device %d, not %d", A->dev, dev);
    if (!A->n) return VEXB_OK;
    VEXB_CHECK(x && y, "null vector");
    DeviceGuard g(dev); VEXB_CHECK(g.ok, "cannot select device %d", dev);
    cudaStream_t st = (cudaStream_t)stream;
    if (param("ccsr.jit", CCSR_DEFAULT_JIT)) {
        bool done = false;
        vexb_ccsr *M = const_cast<vexb_ccsr *>(A);                    // lazily attaches the specialised kernel
        if (A->val_dtype == VEXB_F64) VEXB_TRY(launch_jit<double>(M, st, (const double *)x, (double *)y, alpha, append, &done));
        else VEXB_TRY(launch_jit<float>(M, st, (const float *)x, (float *)y, (float)alpha, append, &done));
        if (done) return VEXB_OK;
    }
    if (A->val_dtype == VEXB_F64) return launch_idx<double>(A, st, (const double *)x, (double *)y, alpha, append);
    return launch_idx<float>(A, st, (const float *)x, (float *)y, (float)alpha, append);
}

extern "C" int vexb_ccsr_jit_source(size_t m, const int32_t *row, const int32_t *col, const void *val, int val_dtype,
                                    int idx_bytes, char *buf, size_t *len, int compile) {
    VEXB_CHECK(len && row, "null argument");
    VEXB_CHECK(val_dtype == VEXB_F64 || val_dtype == VEXB_F32, "CCSR values must be float or double");
    VEXB_CHECK(idx_bytes == 1 || idx_bytes == 2 || idx_bytes == 4, "idx_bytes must be 1, 2 or 4");
    VEXB_CHECK(m >= 1 && m <= CCSR_JIT_MAX_ROWS && row[0] == 0 && row[m] >= 0 && (size_t)row[m] <= CCSR_JIT_MAX_NNZ,
               "table too large for a specialised kernel (at most %zu unique rows, %zu entries)", CCSR_JIT_MAX_ROWS, CCSR_JIT_MAX_NNZ);
    std::vector<int> hrow(row, row + m + 1), hcol(col, col + row[m]);
    std::vector<double> hval((size_t)row[m]);
    for (int j = 0; j < row[m]; ++j) hval[(size_t)j] = val_dtype == VEXB_F64 ? ((const double *)val)[j] : (double)((const float *)val)[j];
    return jit_print(ccsr_jit_source(val_dtype, idx_bytes, hrow, hcol, hval), compile, false, buf, len);
}
