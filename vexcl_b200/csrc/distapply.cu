// SpMat::apply as ONE kernel per GPU, with the halo pushed through NVLink peer memory.
//
// Replaces vexcl/spmat.hpp:120-185 (gather -> D2H -> host shuffle -> H2D -> local product -> remote product, three host
// synchronisations) and this library's own NCCL path (pack kernel, grouped ncclSend/ncclRecv kernel, interior kernel,
// two boundary kernels, a stream fork and join: five launches and the NCCL latency per product).  At 8 GPUs the named
// strong-scaling configurations leave only tens of microseconds of HBM time per product, so the launches and the message
// latency ARE the product; here a product is one launch:
//
//   blocks [0, P)        push: gather x[send_cols] and store the values straight into the ghost buffers of the GPUs that
//                        need them (plain stores to peer-mapped memory), then publish an epoch flag there with a
//                        system-scope release store;
//   blocks [P, P+B)      boundary rows: local entries first, then wait (acquire loads on the flags in my own memory) until
//                        every neighbour's values for this epoch have landed, then  y = alpha*sum_local (+ y);
//                        y += alpha*sum_remote  -- the order of csr.inl:188-209 (mul_local then mul_remote), so the bits
//                        match the unfused path;
//   blocks [P+B, ...)    interior rows (no ghost entries): the hybrid-ELL row body of hell_kernel (a row per thread) or
//                        the sliced-ELL body of sell_kernel (a slice per warp), untouched by the halo.
//
// Blocks are dispatched in index order: pushes leave first; the few boundary blocks come next and sit out the NVLink
// round trip while the interior rows keep the SMs busy.  Ghost buffers and flags are double-buffered by epoch parity and protected by
// acknowledgements (a sender waits until the receiver has finished reading what it pushed two epochs ago), the epoch
// lives in device memory and is advanced by the kernel itself, so the launch is CUDA-graph replayable.  A neighbour
// that never shows up makes the waiters give up after ~20 s: they write NaN into the rows they could not compute and
// raise the process-wide peer fault (vexb_peer_fault), instead of hanging or folding stale values.
//
// Optionally the kernel also accumulates dot(dot_with, y_new) over the rows it produces: every block leaves one partial,
// and a one-block second launch (dot_fold_kernel) folds them in a fixed order and combines the value across the GPUs
// through the reduction mailboxes of peer.cuh.  That is q = A p and (p, q) of a CG iteration without re-reading p and q
// (sparse/product.hpp:45-130 is the reference's fused form on one device).
#include "dspmat.hpp"
#include "spmv_dev.cuh"
#include "peer.cuh"
#include <algorithm>

namespace vexb {

constexpr int kHaloHeaderWords = 128;            // 1 KB header, then the two ghost buffers
constexpr int kHaloArrive = 32, kHaloAck = 64;   // word offsets: arrive[parity*16 + src], ack[parity*16 + dst]
constexpr int kPushChunk = 1024;                 // values per push block (256 threads x 4)

struct HaloLink {
    int dev = 0, rank = 0, nparts = 1;
    unsigned long long *box = nullptr;                       // mine: header + 2 x n_ghost values
    size_t box_bytes = 0;
    unsigned long long *peers[VEXB_MAX_PEERS] = {nullptr};   // every part's box as mapped here (NULL = not a neighbour)
    bool ipc_opened[VEXB_MAX_PEERS] = {false};
    int4 *push_blk = nullptr; int n_push_blocks = 0;         // per push block: {dst, first index in send_cols, count, blocks of this dst}
    // boundary rows in mixed ELL form: col >= 0 local x index, col <= -2 ghost index -(col+2), -1 padding
    int *b_col = nullptr; void *b_val = nullptr; int *b_rows = nullptr;
    size_t b_n = 0, b_pitch = 0; int b_w = 0;
    unsigned long long *fault_host = nullptr;                // mapped pinned word shared by the process (peer.cu)
    bool disabled = false;                                   // vexb_dspmat_halo_disconnect: use NCCL / copies
    void *dot_ws = nullptr; size_t dot_ws_bytes = 0;         // per-block partials of the fused dot (allocated at first use)
};

template <class T>
struct DistArgs {
    // halo
    unsigned long long *box[VEXB_MAX_PEERS];
    unsigned long long ghost_stride[VEXB_MAX_PEERS];         // n_ghost of part p (values per parity buffer)
    unsigned long long land_off[VEXB_MAX_PEERS];             // where my values start in part p's ghost buffer
    unsigned int recv_mask, send_mask;
    int rank, nparts;
    const int4 *push_blk; const int *send_cols; int n_push_blocks;
    // interior strip (hybrid ELL)
    size_t n_int, pitch; int w_dyn; EllShifts shift; const void *ell_col /* vexb_spmat::ell_col_any() */; const T *ell_val /* ell_val_any() */;
    const int *tail_ptr, *tail_col; const T *tail_val; const int *int_row_ids; size_t y_off; int n_int_blocks;
    // boundary rows
    size_t b_n, b_pitch; int b_w; const int *b_col; const T *b_val; const int *b_rows; int n_bnd_blocks;
    const T *x; T *y; T alpha; int append;
    // optional dot(dot_with, y_new)
    const T *dot_with; T *dot_result; void *dot_ws; PeerArgs pa;
    unsigned long long *fault_host;
    // interior strip (sliced ELL): what sell_kernel takes; int_row_ids and y_off as above.  Last, so that the hybrid-ELL
    // instantiations read every other field where they did before.
    size_t n_slices; const int *sell_ptr, *sell_perm; const void *sell_col; const T *sell_val; int sell_shift;
};

template <class T> __device__ __forceinline__ T nan_of();
template <> __device__ __forceinline__ double nan_of<double>() { return __longlong_as_double(0x7ff8000000000000ll); }
template <> __device__ __forceinline__ float nan_of<float>() { return __int_as_float(0x7fc00000); }

__device__ __forceinline__ unsigned long long globaltimer_ns() {
    unsigned long long t; asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t)); return t;
}

// Spin until *flag >= want (acquire, system scope).  Returns false after ~20 s.
__device__ __forceinline__ bool wait_flag(const unsigned long long *flag, unsigned long long want) {
    if (ld_acquire_sys(flag) >= want) return true;
    const unsigned long long t0 = globaltimer_ns();
    for (unsigned it = 0;; ++it) {
        if (ld_acquire_sys(flag) >= want) return true;
        __nanosleep(it < 64 ? 32 : 256);
        if ((it & 1023u) == 1023u && globaltimer_ns() - t0 > 20000000000ull) return false;
    }
}

// Column type of a sliced-ELL interior strip: dist_apply_kernel<T, 0, SellCol<C>, DOT> runs sell_kernel's body on it
// (C = short: 16-bit offsets from (row + sell_shift), C = int: the columns).
template <class C> struct SellCol {};
template <class C> struct sell_col_of { using type = void; };
template <class C> struct sell_col_of<SellCol<C>> { using type = C; };

// Interior block ib of a sliced-ELL strip: 8 slices, one warp per slice and one lane per row, sell_kernel's loop
// restated (4 slots a turn, then the rest one by one, products added in storage order, the same cache hints), so every
// row gets the bits sell_kernel gives it.  Returns the lane's term of dot(dot_with, y_new); a padding lane (perm -1) and
// a warp past the last slice write nothing and return +0, as a thread past the last row of the hybrid-ELL body does.
template <class T, class C, bool DOT>
__device__ __forceinline__ T dist_sell_rows(const DistArgs<T> &a, size_t ib) {
    const size_t s = ib * 8 + (threadIdx.x >> 5);
    if (s >= a.n_slices) return T(0);
    const int lane = threadIdx.x & 31;
    const uint64_t stream = l2_policy_stream(), keep = l2_policy_keep();
    const int base = __ldg(a.sell_ptr + s), w = (__ldg(a.sell_ptr + s + 1) - base) >> 5;
    const int r = ldg_stream(a.sell_perm + s * 32 + lane, stream);
    const C *cp = (const C *)a.sell_col + base + lane;
    const T *vp = a.sell_val + base + lane;
    const size_t rr = r >= 0 ? (size_t)r : 0;
    T sum = T(0);
    int k = 0;
    for (; k + 4 <= w; k += 4) {
        int c[4]; T v[4], xv[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) { c[u] = ell_column(ldg_stream(cp + (k + u) * 32, stream), rr, a.sell_shift); v[u] = ldg_stream(vp + (k + u) * 32, stream); }
#pragma unroll
        for (int u = 0; u < 4; ++u) xv[u] = c[u] != -1 ? ldg_keep(a.x + c[u], keep) : T(0);
#pragma unroll
        for (int u = 0; u < 4; ++u) if (c[u] != -1) sum = t_add<T>(sum, t_mul<T>(v[u], xv[u]));
    }
    for (; k < w; ++k) {
        const int c = ell_column(ldg_stream(cp + k * 32, stream), rr, a.sell_shift);
        const T v = ldg_stream(vp + k * 32, stream);
        if (c != -1) sum = t_add<T>(sum, t_mul<T>(v, ldg_keep(a.x + c, keep)));
    }
    if (r < 0) return T(0);
    const size_t ry = a.y_off + (a.int_row_ids ? (size_t)a.int_row_ids[r] : (size_t)r);
    const T v = t_mul<T>(a.alpha, sum);
    const T out = a.append ? t_add<T>(a.y[ry], v) : v;
    a.y[ry] = out;
    return DOT ? t_mul<T>(a.dot_with[ry], out) : T(0);
}

// dot partials: one value per block in dot_ws (own buffer, not the Reductor workspace)
// Register bound: 32 per thread (8 blocks per SM).  Row-class strips get 40 (6 blocks per SM): under 32 their row body,
// which keeps all W gathers of x in flight before the class byte returns (hell_class_rows), spilled 24 bytes at every
// width, in the interior rows as well as the boundary rows.
// C = SellCol<short | int>: the interior strip is sliced ELL (dist_sell_rows), W is 0.  In double those spilled 44 bytes
// under 32 registers (4 slots of 8-byte values and gathers in flight beside the boundary rows' state) and get 40 (6 blocks
// per SM) as well; in float they fit 32.
template <class T, class C> constexpr int dist_min_blocks() {
    return std::is_same<C, EllClass>::value || (!std::is_void<typename sell_col_of<C>::type>::value && sizeof(T) == 8) ? 6 : 8;
}
template <class T, int W, class C, bool DOT>
__global__ void __launch_bounds__(256, dist_min_blocks<T, C>()) dist_apply_kernel(const __grid_constant__ DistArgs<T> a) {
    unsigned long long *mine = a.box[a.rank];
    __shared__ unsigned long long s_epoch;
    __shared__ int s_ok;
    const int b = blockIdx.x;
    // Block order: push, boundary rows, interior rows.  Boundary blocks are few and their life is a chain of memory round
    // trips (local entries, wait for the neighbours' flags, ghost entries); dispatched last -- as in the first version --
    // that chain is the tail of the kernel.  Dispatched right after the push blocks they wait while the interior rows keep
    // the SMs busy.
    // Only push and boundary blocks take part in the epoch protocol; interior blocks never look at it.
    const bool halo_block = b < a.n_push_blocks + a.n_bnd_blocks;
    if (halo_block) {
        if (threadIdx.x == 0) { s_epoch = ld_relaxed_sys(mine) + 1; s_ok = 1; }
        __syncthreads();
    }
    const unsigned long long e = halo_block ? s_epoch : 0ull;
    const int parity = (int)(e & 1ull);
    T dot_acc = T(0);

    if (b < a.n_push_blocks) {
        // ---- push my x values into the neighbours' ghost buffers ----
        const int4 pb = a.push_blk[b];                       // {dst, begin, count, blocks of dst}
        const int dst = pb.x;
        if (threadIdx.x == 0 && e > 2) {
            // the receiver must have finished reading what I pushed two epochs ago (same parity buffer)
            if (!wait_flag(mine + kHaloAck + parity * VEXB_MAX_PEERS + dst, e - 2)) s_ok = 0;
        }
        __syncthreads();
        T *ghost = reinterpret_cast<T *>(a.box[dst] + kHaloHeaderWords) + (size_t)parity * a.ghost_stride[dst] + a.land_off[dst];
        const int lo = pb.y, cnt = pb.z;
        const int *cols = a.send_cols + lo;
        // position within this destination's segment: push_blk.y is an index into send_cols; the segment of dst starts at seg0
        const int seg0 = a.push_blk[b - (int)((unsigned)pb.w >> 16)].y;      // first block of this dst (offset stored in the high half)
        for (int i = threadIdx.x; i < cnt; i += blockDim.x) ghost[(lo - seg0) + i] = __ldg(a.x + cols[i]);
        __threadfence_system();
        __syncthreads();
        if (threadIdx.x == 0) {
            if (!s_ok) { mine[1] = e; if (a.fault_host) *a.fault_host = e; }
            const int nblk = pb.w & 0xffff;
            unsigned int *cnt_p = reinterpret_cast<unsigned int *>(mine + 8) + dst;
            const unsigned int old = atomicAdd(cnt_p, 1u);
            if (old == (unsigned)nblk - 1) {
                *cnt_p = 0;
                __threadfence_system();
                st_release_sys(a.box[dst] + kHaloArrive + parity * VEXB_MAX_PEERS + a.rank, e);
            }
        }
    } else if (b >= a.n_push_blocks + a.n_bnd_blocks) {
        // ---- interior rows ----
        using SC = typename sell_col_of<C>::type;
        const size_t i = (size_t)(b - a.n_push_blocks - a.n_bnd_blocks) * blockDim.x + threadIdx.x;
        if constexpr (!std::is_void<SC>::value) {
            dot_acc = dist_sell_rows<T, SC, DOT>(a, (size_t)(b - a.n_push_blocks - a.n_bnd_blocks));
        } else if (i < a.n_int) {
            const uint64_t stream = l2_policy_stream(), keep = l2_policy_keep();
            const T sum = hell_row_sum<T, W, C>(i, a.pitch, a.w_dyn, (const C *)a.ell_col, a.shift, a.ell_val, a.tail_ptr, a.tail_col,
                                                a.tail_val, a.x, stream, keep);
            const size_t r = a.int_row_ids ? (size_t)a.int_row_ids[i] : a.y_off + i;
            const T v = t_mul<T>(a.alpha, sum);
            const T out = a.append ? t_add<T>(a.y[r], v) : v;
            a.y[r] = out;
            if (DOT) dot_acc = t_mul<T>(a.dot_with[r], out);
        }
    } else {
        // ---- boundary rows: local entries first, then -- once the halo has landed -- the ghost entries ----
        const size_t i = (size_t)(b - a.n_push_blocks) * blockDim.x + threadIdx.x;
        const bool live = i < a.b_n;
        T sloc = T(0);
        const uint64_t keep = l2_policy_keep();
        if (live) {
            // four slots at a time: the column loads, then the value loads and gathers travel together (a plain loop is
            // 2 * b_w dependent round trips); products still added in slot order
            for (int k0 = 0; k0 < a.b_w; k0 += 4) {
                int c[4]; T v[4], xv[4];
#pragma unroll
                for (int u = 0; u < 4; ++u) c[u] = k0 + u < a.b_w ? a.b_col[i + (size_t)(k0 + u) * a.b_pitch] : -1;
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    v[u] = c[u] >= 0 ? a.b_val[i + (size_t)(k0 + u) * a.b_pitch] : T(0);
                    xv[u] = c[u] >= 0 ? ldg_keep(a.x + c[u], keep) : T(0);
                }
#pragma unroll
                for (int u = 0; u < 4; ++u) if (c[u] >= 0) sloc = t_add<T>(sloc, t_mul<T>(v[u], xv[u]));
            }
        }
        if ((int)threadIdx.x < a.nparts && ((a.recv_mask >> threadIdx.x) & 1u)) {
            if (!wait_flag(mine + kHaloArrive + parity * VEXB_MAX_PEERS + threadIdx.x, e)) {
                atomicExch(&s_ok, 0);
                mine[1] = e; if (a.fault_host) *a.fault_host = e;
            }
        }
        __syncthreads();
        if (live) {
            const size_t r = (size_t)a.b_rows[i];
            T out;
            if (s_ok) {
                const T *ghost = reinterpret_cast<const T *>(mine + kHaloHeaderWords) + (size_t)parity * a.ghost_stride[a.rank];
                T srem = T(0);
                for (int k0 = 0; k0 < a.b_w; k0 += 4) {
                    int c[4]; T v[4], gv[4];
#pragma unroll
                    for (int u = 0; u < 4; ++u) c[u] = k0 + u < a.b_w ? a.b_col[i + (size_t)(k0 + u) * a.b_pitch] : -1;
#pragma unroll
                    for (int u = 0; u < 4; ++u) {
                        v[u] = c[u] <= -2 ? a.b_val[i + (size_t)(k0 + u) * a.b_pitch] : T(0);
                        // written by another GPU during this kernel: bypass L1 (volatile is enough after the acquire)
                        gv[u] = c[u] <= -2 ? *reinterpret_cast<const volatile T *>(ghost + (-(c[u] + 2))) : T(0);
                    }
#pragma unroll
                    for (int u = 0; u < 4; ++u) if (c[u] <= -2) srem = t_add<T>(srem, t_mul<T>(v[u], gv[u]));
                }
                const T v = t_mul<T>(a.alpha, sloc);
                out = a.append ? t_add<T>(a.y[r], v) : v;
                out = t_add<T>(out, t_mul<T>(a.alpha, srem));
            } else out = nan_of<T>();
            a.y[r] = out;
            if (DOT) dot_acc = t_mul<T>(a.dot_with[r], out);
        }
        __syncthreads();
        if (threadIdx.x == 0 && a.n_bnd_blocks > 0) {
            unsigned int *done = reinterpret_cast<unsigned int *>(mine + 3);
            const unsigned int old = atomicAdd(done, 1u);
            if (old == (unsigned)a.n_bnd_blocks - 1) {
                *done = 0;
                __threadfence_system();
                // every boundary block has read its ghosts: the senders may reuse this parity buffer
                for (int p = 0; p < a.nparts; ++p)
                    if ((a.recv_mask >> p) & 1u) st_release_sys(a.box[p] + kHaloAck + parity * VEXB_MAX_PEERS + a.rank, e);
            }
        }
    }

    // ---- block epilogue: the epoch advances when the last halo block is done (they all read it at their start); with
    //      DOT every block leaves its partial of dot(dot_with, y) for dot_fold_kernel (no fence, no ticket: the blocks
    //      are short, a memory round trip at the end of each would cost a quarter of the kernel) ----
    if (halo_block && threadIdx.x == 0) {
        unsigned int *ticket = reinterpret_cast<unsigned int *>(mine + 2);
        const unsigned int old = atomicAdd(ticket, 1u);
        if (old == (unsigned)(a.n_push_blocks + a.n_bnd_blocks) - 1) { *ticket = 0; mine[0] = e; }
    }
    if (!DOT) return;
    __shared__ T s_part[8];
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) dot_acc = t_add<T>(dot_acc, __shfl_down_sync(0xffffffffu, dot_acc, off));
    if ((threadIdx.x & 31) == 0) s_part[threadIdx.x >> 5] = dot_acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        T tot = s_part[0];
        for (int w = 1; w < 8; ++w) tot = t_add<T>(tot, s_part[w]);
        reinterpret_cast<T *>(a.dot_ws)[b] = tot;
    }
}

// Second (one-block) launch of a product + dot: folds the per-block partials in a fixed order (thread t takes partials
// t, t + 1024, ...; then shuffle trees), combines the value across the GPUs through the reduction mailboxes (peer.cuh) and
// stores it.  Every GPU ends with the same bits.
template <class T>
__global__ void __launch_bounds__(1024) dot_fold_kernel(const T *__restrict__ parts, unsigned int n, T *result, PeerArgs pa,
                                                         unsigned long long *fault_host) {
    __shared__ T s_part[32];
    // thread t adds partials t, t + 1024, ... in that order; the loads of 16 of them travel together (a plain loop waits
    // for memory once per partial)
    T g = T(0);
    for (unsigned int k0 = threadIdx.x; k0 < n; k0 += 16u * blockDim.x) {
        T v[16];
#pragma unroll
        for (int u = 0; u < 16; ++u) { const unsigned int k = k0 + (unsigned)u * blockDim.x; v[u] = k < n ? parts[k] : T(0); }
#pragma unroll
        for (int u = 0; u < 16; ++u) { const unsigned int k = k0 + (unsigned)u * blockDim.x; if (k < n) g = t_add<T>(g, v[u]); }
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) g = t_add<T>(g, __shfl_down_sync(0xffffffffu, g, off));
    if ((threadIdx.x & 31) == 0) s_part[threadIdx.x >> 5] = g;
    __syncthreads();
    if (threadIdx.x < 32) {
        g = s_part[threadIdx.x];
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) g = t_add<T>(g, __shfl_down_sync(0xffffffffu, g, off));
        if (threadIdx.x == 0) s_part[0] = g;
    }
    __syncthreads();
    if (pa.nranks > 1) {
        __shared__ unsigned long long px[VEXB_MAX_PEERS], py[VEXB_MAX_PEERS];
        unsigned long long bits = 0; { T t0 = s_part[0]; memcpy(&bits, &t0, sizeof(T)); }
        const bool ok = peer_exchange(pa, bits, 0ull, px, py);
        if (threadIdx.x == 0) {
            T tot; memcpy(&tot, &px[0], sizeof(T));
            for (int r = 1; r < pa.nranks; ++r) { T v; memcpy(&v, &px[r], sizeof(T)); tot = t_add<T>(tot, v); }
            s_part[0] = ok ? tot : nan_of<T>();
            if (!ok && fault_host) *fault_host = ~0ull;
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) result[0] = s_part[0];
}

} // namespace vexb

using namespace vexb;

void vexb::halo_link_destroy(HaloLink *h) {
    if (!h) return;
    DeviceGuard g(h->dev);
    for (int p = 0; p < h->nparts; ++p) if (h->ipc_opened[p]) cudaIpcCloseMemHandle(h->peers[p]);
    cudaFree(h->box); cudaFree(h->push_blk); cudaFree(h->b_col); cudaFree(h->b_val); cudaFree(h->b_rows); cudaFree(h->dot_ws);
    delete h;
}

namespace vexb { unsigned long long *peer_fault_word(); }

// Allocate the box and the push table; boundary rows come from dspmat_create (dspmat.cu fills b_* through halo_set_boundary).
int vexb::halo_prepare(vexb_dspmat *A) {
    if (A->halo) return VEXB_OK;
    VEXB_CHECK(A->nparts <= VEXB_MAX_PEERS, "peer-memory halo supports at most %d parts", VEXB_MAX_PEERS);
    size_t n_send = 0;
    for (size_t c : A->send_counts) n_send += c;
    VEXB_CHECK(n_send < (size_t)INT32_MAX && A->n_ghost < (size_t)INT32_MAX, "halo too large");
    DeviceGuard g(A->dev); VEXB_CHECK(g.ok, "cannot select device %d", A->dev);
    auto *h = new HaloLink();
    h->dev = A->dev; h->rank = A->part; h->nparts = A->nparts;
    const size_t vs = dtype_size(A->val_dtype);
    h->box_bytes = (size_t)kHaloHeaderWords * 8 + 2 * std::max<size_t>(A->n_ghost, 1) * vs;
    cudaError_t e = cudaMalloc((void **)&h->box, h->box_bytes);
    if (e != cudaSuccess) { delete h; VEXB_FAIL(VEXB_ERR_CUDA, "cudaMalloc of the halo box failed: %s", cudaGetErrorString(e)); }
    cudaMemset(h->box, 0, h->box_bytes);
    h->peers[h->rank] = h->box;
    // push blocks: chunks of kPushChunk values, never straddling two destinations.  w = (offset of this block within its
    // destination's run of blocks) << 16 | number of blocks of that destination
    std::vector<int4> blk;
    size_t so = 0;
    for (int p = 0; p < A->nparts; ++p) {
        const size_t cnt = A->send_counts[p];
        const int nb = (int)((cnt + kPushChunk - 1) / kPushChunk);
        if (nb > 0x7fff) { halo_link_destroy(h); VEXB_FAIL(VEXB_ERR_UNSUPPORTED, "halo segment of %zu values is too large for the peer-memory path", cnt); }
        for (int k = 0; k < nb; ++k) {
            const size_t lo = so + (size_t)k * kPushChunk;
            blk.push_back(make_int4(p, (int)lo, (int)std::min<size_t>(kPushChunk, so + cnt - lo), (k << 16) | nb));
        }
        so += cnt;
    }
    h->n_push_blocks = (int)blk.size();
    if (!blk.empty()) {
        e = cudaMalloc((void **)&h->push_blk, blk.size() * sizeof(int4));
        if (e == cudaSuccess) e = cudaMemcpy(h->push_blk, blk.data(), blk.size() * sizeof(int4), cudaMemcpyHostToDevice);
        if (e != cudaSuccess) { halo_link_destroy(h); VEXB_FAIL(VEXB_ERR_CUDA, "push table upload failed: %s", cudaGetErrorString(e)); }
    }
    h->fault_host = peer_fault_word();
    cudaDeviceSynchronize();
    A->halo = h;
    return VEXB_OK;
}

namespace vexb {
// Called by vexb_dspmat_create: the boundary rows (every row outside the interior strip) in mixed ELL form.
int halo_set_boundary(vexb_dspmat *A, const std::vector<int> &rows, int width, const std::vector<int> &col, const void *val) {
    VEXB_TRY(halo_prepare(A));
    HaloLink *h = A->halo;
    DeviceGuard g(A->dev);
    const size_t vs = dtype_size(A->val_dtype);
    h->b_n = rows.size(); h->b_w = width; h->b_pitch = (rows.size() + 15) / 16 * 16;
    if (!h->b_n) return VEXB_OK;
    VEXB_CUDA(cudaMalloc((void **)&h->b_rows, h->b_n * 4));
    VEXB_CUDA(cudaMemcpy(h->b_rows, rows.data(), h->b_n * 4, cudaMemcpyHostToDevice));
    if (width > 0) {
        VEXB_CUDA(cudaMalloc((void **)&h->b_col, col.size() * 4));
        VEXB_CUDA(cudaMemcpy(h->b_col, col.data(), col.size() * 4, cudaMemcpyHostToDevice));
        VEXB_CUDA(cudaMalloc(&h->b_val, col.size() * vs));
        VEXB_CUDA(cudaMemcpy(h->b_val, val, col.size() * vs, cudaMemcpyHostToDevice));
    }
    return VEXB_OK;
}
}

extern "C" int vexb_dspmat_halo_handle(vexb_dspmat *A, void *handle64) {
    VEXB_CHECK(A && handle64, "NULL argument");
    VEXB_TRY(halo_prepare(A));
    DeviceGuard g(A->dev);
    cudaIpcMemHandle_t hd;
    VEXB_CUDA(cudaIpcGetMemHandle(&hd, A->halo->box));
    memcpy(handle64, &hd, sizeof(hd));
    return VEXB_OK;
}

// A part needs the boxes of the parts it sends to (ghost buffers, arrival flags) and receives from (acknowledgements).
static bool is_neighbour(const vexb_dspmat *A, int p) { return p != A->part && (A->send_counts[p] || A->recv_counts[p]); }

extern "C" int vexb_dspmat_halo_connect(vexb_dspmat *A, const void *handles) {
    VEXB_CHECK(A && handles, "NULL argument");
    if (A->values_f32) VEXB_FAIL(VEXB_ERR_UNSUPPORTED, "no peer-memory halo for float values (VEXB_FMT_VALUES_F32): NCCL or copies");
    VEXB_TRY(halo_prepare(A));
    HaloLink *h = A->halo;
    DeviceGuard g(A->dev); VEXB_CHECK(g.ok, "cannot select device %d", A->dev);
    for (int p = 0; p < A->nparts; ++p) {
        if (!is_neighbour(A, p) || h->peers[p]) continue;
        cudaIpcMemHandle_t hd;
        memcpy(&hd, (const char *)handles + (size_t)p * VEXB_IPC_HANDLE_BYTES, sizeof(hd));
        void *ptr = nullptr;
        VEXB_CUDA(cudaIpcOpenMemHandle(&ptr, hd, cudaIpcMemLazyEnablePeerAccess));
        h->peers[p] = (unsigned long long *)ptr; h->ipc_opened[p] = true;
    }
    return VEXB_OK;
}

extern "C" int vexb_dspmat_halo_connect_local(int nlocal, vexb_dspmat *const *parts) {
    VEXB_CHECK(nlocal >= 1 && parts, "bad arguments");
    VEXB_CHECK(nlocal == parts[0]->nparts, "every part must be local (%d of %d given)", nlocal, parts[0]->nparts);
    for (int a = 0; a < nlocal; ++a)
        if (parts[a] && parts[a]->values_f32) VEXB_FAIL(VEXB_ERR_UNSUPPORTED, "no peer-memory halo for float values (VEXB_FMT_VALUES_F32): NCCL or copies");
    for (int a = 0; a < nlocal; ++a) {
        VEXB_CHECK(parts[a] && parts[a]->part == a, "parts must be passed in order");
        for (int b = a + 1; b < nlocal; ++b) VEXB_CHECK(parts[a]->dev != parts[b]->dev, "the peer-memory halo needs distinct devices");
    }
    for (int a = 0; a < nlocal; ++a) {
        VEXB_TRY(halo_prepare(parts[a]));
        DeviceGuard g(parts[a]->dev);
        for (int b = 0; b < nlocal; ++b) if (is_neighbour(parts[a], b)) {
            int can = 0;
            VEXB_CUDA(cudaDeviceCanAccessPeer(&can, parts[a]->dev, parts[b]->dev));
            if (!can) VEXB_FAIL(VEXB_ERR_UNSUPPORTED, "device %d cannot access device %d", parts[a]->dev, parts[b]->dev);
            cudaError_t e = cudaDeviceEnablePeerAccess(parts[b]->dev, 0);
            if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) VEXB_CUDA(e);
            cudaGetLastError();
        }
    }
    for (int a = 0; a < nlocal; ++a) for (int b = 0; b < nlocal; ++b) if (is_neighbour(parts[a], b)) parts[a]->halo->peers[b] = parts[b]->halo->box;
    return VEXB_OK;
}

extern "C" int vexb_dspmat_halo_disconnect(vexb_dspmat *A) {
    VEXB_CHECK(A, "NULL argument");
    if (!A->halo) return VEXB_OK;
    DeviceGuard g(A->dev);
    for (int p = 0; p < A->nparts; ++p) {
        if (p == A->part) continue;
        if (A->halo->ipc_opened[p]) cudaIpcCloseMemHandle(A->halo->peers[p]);
        A->halo->peers[p] = nullptr; A->halo->ipc_opened[p] = false;
    }
    A->halo->disabled = true;
    return VEXB_OK;
}

extern "C" int vexb_dspmat_halo_connected(const vexb_dspmat *A, int *connected) {
    VEXB_CHECK(A && connected, "NULL argument");
    bool ok = A->halo != nullptr && !A->halo->disabled;
    for (int p = 0; ok && p < A->nparts; ++p) if (is_neighbour(A, p) && !A->halo->peers[p]) ok = false;
    *connected = ok ? 1 : 0;
    return VEXB_OK;
}

namespace vexb {

template <class T, bool DOT>
static int launch_dist(const vexb_dspmat *A, cudaStream_t st, const DistArgs<T> &a, unsigned grid) {
    const vexb_spmat *S = A->loc;
    const bool hell = S && S->fmt == VEXB_FMT_HELL && a.n_int_blocks > 0;
    const bool sell = S && S->fmt == VEXB_FMT_SELL && a.n_int_blocks > 0;
    const size_t w = hell ? S->ell_width : 0;
#define DL(W) do { if (hell && S->ell_col16) dist_apply_kernel<T, W, short, DOT><<<grid, 256, 0, st>>>(a); \
                   else dist_apply_kernel<T, W, int, DOT><<<grid, 256, 0, st>>>(a); } while (0)
    if (sell) {
        if (S->sell_col16) dist_apply_kernel<T, 0, SellCol<short>, DOT><<<grid, 256, 0, st>>>(a);
        else dist_apply_kernel<T, 0, SellCol<int>, DOT><<<grid, 256, 0, st>>>(a);
    } else if (hell && S->ell_class) {
        switch (w) {   // = the widths spmv.cu build() gives row classes
            case 5: dist_apply_kernel<T, 5, EllClass, DOT><<<grid, 256, 0, st>>>(a); break;
            case 7: dist_apply_kernel<T, 7, EllClass, DOT><<<grid, 256, 0, st>>>(a); break;
            case 3: dist_apply_kernel<T, 3, EllClass, DOT><<<grid, 256, 0, st>>>(a); break;
            default: VEXB_FAIL(VEXB_ERR_UNSUPPORTED, "no dist_apply_kernel for row classes of width %zu", w);
        }
    } else if (hell && S->ell_mask) {
        switch (w) {   // = the widths spmv.cu build() gives slot masks
            case 5: dist_apply_kernel<T, 5, EllDiag, DOT><<<grid, 256, 0, st>>>(a); break;
            case 7: dist_apply_kernel<T, 7, EllDiag, DOT><<<grid, 256, 0, st>>>(a); break;
            case 3: dist_apply_kernel<T, 3, EllDiag, DOT><<<grid, 256, 0, st>>>(a); break;
            default: VEXB_FAIL(VEXB_ERR_UNSUPPORTED, "no dist_apply_kernel for slot masks of width %zu", w);
        }
    } else switch (w) {
        case 5: DL(5); break; case 7: DL(7); break; case 3: DL(3); break; case 9: DL(9); break;   // = ell_width_is_unrolled_everywhere
        default: DL(0); break;
    }
#undef DL
    VEXB_LAUNCHED();
    return VEXB_OK;
}

// y (=|+=) alpha * A x for one part through the peer-memory halo.  If the interior strip is hybrid or sliced ELL (with
// entries) everything is one launch; otherwise the interior runs as its own kernel on `st` and push + boundary rows follow
// in a second launch on the part's side stream (forked from / joined to `st` with events, so the pair is still
// graph-capturable).
template <class T>
static int dist_apply_t(const vexb_dspmat *A, cudaStream_t st, const T *x, T *y, T alpha, int append, const T *dot_with,
                        T *dot_result, const vexb_peer *peer) {
    HaloLink *h = A->halo;
    DistArgs<T> a; memset(&a, 0, sizeof(a));
    for (int p = 0; p < A->nparts; ++p) {
        a.box[p] = h->peers[p];
        a.ghost_stride[p] = A->ghost_counts[p];
        a.land_off[p] = A->land_off[p];
        if (p != A->part && A->recv_counts[p]) a.recv_mask |= 1u << p;
        if (p != A->part && A->send_counts[p]) a.send_mask |= 1u << p;
    }
    a.rank = A->part; a.nparts = A->nparts;
    a.push_blk = h->push_blk; a.send_cols = A->send_cols; a.n_push_blocks = h->n_push_blocks;
    a.b_n = h->b_n; a.b_pitch = h->b_pitch; a.b_w = h->b_w; a.b_col = h->b_col; a.b_val = (const T *)h->b_val; a.b_rows = h->b_rows;
    a.n_bnd_blocks = (int)((h->b_n + 255) / 256);
    a.x = x; a.y = y; a.alpha = alpha; a.append = append;
    a.dot_with = dot_with; a.dot_result = dot_result;
    memset(&a.pa, 0, sizeof(a.pa));
    if (peer && peer->nranks > 1) a.pa = peer->args();
    a.fault_host = h->fault_host;
    const vexb_spmat *S = A->loc;
    // an interior strip without entries keeps the second path: its product only zeroes y (spmv_launch)
    const bool hell_interior = S && S->fmt == VEXB_FMT_HELL && S->nnz > 0 && S->nrows_stored > 0;
    const bool sell_interior = S && S->fmt == VEXB_FMT_SELL && S->nnz > 0 && S->nrows_stored > 0;
    const bool fused_interior = hell_interior || sell_interior;
    if (hell_interior) {
        a.n_int = S->nrows_stored; a.pitch = S->ell_pitch; a.w_dyn = (int)S->ell_width; a.shift = S->ell_shifts;
        a.ell_col = S->ell_col_any(); a.ell_val = (const T *)S->ell_val_any();
        a.tail_ptr = S->tail_ptr; a.tail_col = S->tail_col; a.tail_val = (const T *)S->tail_val;
        a.int_row_ids = S->row_ids; a.y_off = S->y_offset;
        a.n_int_blocks = (int)((S->nrows_stored + 255) / 256);
    } else if (sell_interior) {
        a.n_slices = S->n_slices; a.sell_ptr = S->sell_ptr; a.sell_perm = S->sell_perm;
        a.sell_col = S->sell_col16 ? (const void *)S->sell_col16 : (const void *)S->sell_col; a.sell_val = (const T *)S->sell_val;
        a.sell_shift = S->sell_col16 ? S->sell_shift : 0;
        a.int_row_ids = S->row_ids; a.y_off = S->y_offset;
        a.n_int_blocks = (int)((S->n_slices + 7) / 8);                // 8 slices per block, as sell_kernel
    } else if (dot_with) {
        VEXB_FAIL(VEXB_ERR_UNSUPPORTED, "the fused product + dot needs a hybrid- or sliced-ELL interior strip");
    }
    const unsigned grid = (unsigned)(a.n_push_blocks + a.n_int_blocks + a.n_bnd_blocks);
    if (dot_with) {
        const size_t need = (size_t)grid * 8;
        if (h->dot_ws_bytes < need) {                        // first use (outside any graph capture: callers warm up first)
            cudaFree(h->dot_ws); h->dot_ws = nullptr; h->dot_ws_bytes = 0;
            VEXB_CUDA(cudaMalloc(&h->dot_ws, need));
            VEXB_CUDA(cudaMemset(h->dot_ws, 0, need));
            h->dot_ws_bytes = need;
        }
        a.dot_ws = h->dot_ws;
    }
    if (fused_interior) {
        if (grid == 0) return VEXB_OK;
        if (!dot_with) return launch_dist<T, false>(A, st, a, grid);
        VEXB_TRY((launch_dist<T, true>(A, st, a, grid)));
        dot_fold_kernel<T><<<1, 1024, 0, st>>>((const T *)h->dot_ws, grid, dot_result, a.pa, h->fault_host);
        VEXB_LAUNCHED();
        return VEXB_OK;
    }
    // interior as its own kernel (CSR / row patterns / empty), halo + boundary rows beside it
    VEXB_CUDA(cudaEventRecord(A->ev_x, st));
    VEXB_CUDA(cudaStreamWaitEvent(A->side, A->ev_x, 0));
    if (grid) VEXB_TRY((launch_dist<T, false>(A, A->side, a, grid)));
    VEXB_CUDA(cudaEventRecord(A->ev_halo, A->side));
    if (S) VEXB_TRY(vexb_spmv(A->dev, (void *)st, S, x, y, (double)alpha, append));
    VEXB_CUDA(cudaStreamWaitEvent(st, A->ev_halo, 0));
    return VEXB_OK;
}

int dist_apply(const vexb_dspmat *A, cudaStream_t st, const void *x, void *y, double alpha, int append, const void *dot_with,
               void *dot_result, const vexb_peer *peer) {
    DeviceGuard g(A->dev); VEXB_CHECK(g.ok, "cannot select device %d", A->dev);
    if (A->val_dtype == VEXB_F64)
        return dist_apply_t<double>(A, st, (const double *)x, (double *)y, alpha, append, (const double *)dot_with, (double *)dot_result, peer);
    return dist_apply_t<float>(A, st, (const float *)x, (float *)y, (float)alpha, append, (const float *)dot_with, (float *)dot_result, peer);
}

} // namespace vexb
