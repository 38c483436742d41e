// The device side of every reduction: the per-thread fold states (Fold, RtFold), the block and grid finish
// (block_finish) and the one-hop exchange over peer memory that combines the value across GPUs inside the same kernel.
//
// One text serves two compilers.  nvcc includes it into the pre-compiled reductions (csrc/reduce.cu) and the peer
// helpers (csrc/peer.cuh); vexcl_b200/build.py stringifies it byte for byte into the NVRTC programs that reduce
// expressions with user functions or inlined sparse products (csrc/jit.cu, generate_reduce_source), so both kinds of
// kernel fold, finish and combine with the same code.  It therefore includes nothing under NVRTC and uses no host
// library: the program that embeds it defines the VEXB_* reduce-op constants first.
#ifndef VEXB_FOLD_CUH
#define VEXB_FOLD_CUH
#ifndef __CUDACC_RTC__
#include "common.cuh"
#endif

#define VEXB_MAX_PEERS 16

namespace vexb {

template <class T> struct Lim;
template <> struct Lim<double> {
    static __host__ __device__ double lowest() { return -0x1.fffffffffffffp+1023; }
    static __host__ __device__ double highest() { return 0x1.fffffffffffffp+1023; }
};
template <> struct Lim<float> {
    static __host__ __device__ float lowest() { return -0x1.fffffep+127f; }
    static __host__ __device__ float highest() { return 0x1.fffffep+127f; }
};
template <> struct Lim<int> {
    static __host__ __device__ int lowest() { return -2147483647 - 1; }
    static __host__ __device__ int highest() { return 2147483647; }
};
template <> struct Lim<unsigned> {
    static __host__ __device__ unsigned lowest() { return 0u; }
    static __host__ __device__ unsigned highest() { return 4294967295u; }
};
template <> struct Lim<long long> {
    static __host__ __device__ long long lowest() { return -9223372036854775807ll - 1; }
    static __host__ __device__ long long highest() { return 9223372036854775807ll; }
};
template <> struct Lim<unsigned long long> {
    static __host__ __device__ unsigned long long lowest() { return 0ull; }
    static __host__ __device__ unsigned long long highest() { return 18446744073709551615ull; }
};

template <class T> __device__ __forceinline__ T red_add(T a, T b) { return a + b; }
template <> __device__ __forceinline__ double red_add<double>(double a, double b) { return __dadd_rn(a, b); }
template <> __device__ __forceinline__ float red_add<float>(float a, float b) { return __fadd_rn(a, b); }
template <class T> __device__ __forceinline__ T red_sub(T a, T b) { return a - b; }
template <> __device__ __forceinline__ double red_sub<double>(double a, double b) { return __dsub_rn(a, b); }
template <> __device__ __forceinline__ float red_sub<float>(float a, float b) { return __fsub_rn(a, b); }

// Fold state: x (and y for Kahan's compensation / MINMAX's max).
template <int OP, class T> struct Fold {
    T x, y;
    __device__ __forceinline__ void init() {
        if (OP == VEXB_SUM || OP == VEXB_SUM_KAHAN) { x = T(0); y = T(0); }
        else if (OP == VEXB_MAX) { x = Lim<T>::lowest(); y = T(0); }
        else if (OP == VEXB_MIN) { x = Lim<T>::highest(); y = T(0); }
        else { x = Lim<T>::highest(); y = Lim<T>::lowest(); }
    }
    // Same statement order as the reference's per-work-item loops
    // (reductor.hpp:511-533 plain, :537-564 Kahan; ops :60-63, :92-95, :116-119).
    __device__ __forceinline__ void take(T v) {
        if (OP == VEXB_SUM) x = red_add<T>(x, v);
        else if (OP == VEXB_SUM_KAHAN) { const T yy = red_sub<T>(v, y); const T t = red_add<T>(x, yy); y = red_sub<T>(red_sub<T>(t, x), yy); x = t; }
        else if (OP == VEXB_MAX) x = x > v ? x : v;
        else if (OP == VEXB_MIN) x = x < v ? x : v;
        else { x = x < v ? x : v; y = y > v ? y : v; }
    }
    __device__ __forceinline__ void merge(const Fold &o) {
        if (OP == VEXB_SUM || OP == VEXB_SUM_KAHAN) x = red_add<T>(x, o.x);   // tree/host stages are plain adds in the reference too
        else if (OP == VEXB_MAX) x = x > o.x ? x : o.x;
        else if (OP == VEXB_MIN) x = x < o.x ? x : o.x;
        else { x = x < o.x ? x : o.x; y = y > o.y ? y : o.y; }
    }
};

template <int OP, class T>
__device__ __forceinline__ Fold<OP, T> shfl_down_fold(const Fold<OP, T> &f, int off) {
    Fold<OP, T> r;
    r.x = __shfl_down_sync(0xffffffffu, f.x, off);
    r.y = (OP == VEXB_MINMAX) ? __shfl_down_sync(0xffffffffu, f.y, off) : T(0);
    return r;
}

// Several reductions of ONE expression in one pass (vex::CombineReductors, reductor.hpp:132-280): the op is a run-time
// value; every fold then finishes like a single reduction of its op.
template <class T>
struct RtFold {
    T x, y;
    __device__ __forceinline__ void init(int op) {
        x = (op == VEXB_MAX) ? Lim<T>::lowest() : (op == VEXB_MIN) ? Lim<T>::highest() : T(0); y = T(0);
    }
    __device__ __forceinline__ void take(int op, T v) {
        if (op == VEXB_SUM) x = red_add<T>(x, v);
        else if (op == VEXB_SUM_KAHAN) { const T yy = red_sub<T>(v, y); const T t = red_add<T>(x, yy); y = red_sub<T>(red_sub<T>(t, x), yy); x = t; }
        else if (op == VEXB_MAX) x = x > v ? x : v;
        else x = x < v ? x : v;
    }
    __device__ __forceinline__ void merge(int op, const RtFold &o) {
        if (op == VEXB_SUM || op == VEXB_SUM_KAHAN) x = red_add<T>(x, o.x);
        else if (op == VEXB_MAX) x = x > o.x ? x : o.x;
        else x = x < o.x ? x : o.x;
    }
};

struct ReduceWs {               // layout of d_workspace
    unsigned int ticket;        // zero between calls
    unsigned int pad[15];
    // followed by 2 * max_blocks values of 8 bytes
};

template <class T> __device__ __forceinline__ unsigned long long to_bits(T v) { unsigned long long u = 0; memcpy(&u, &v, sizeof(T)); return u; }
template <class T> __device__ __forceinline__ T from_bits(unsigned long long u) { T v; memcpy(&v, &u, sizeof(T)); return v; }

// ---- one-hop all-reduce over NVLink peer memory, callable from inside a kernel ------------------------------------
//
// Every rank owns a small "mailbox" in device memory that all other ranks can write (CUDA IPC mapping
// between processes, peer access inside one process).  To combine one value per rank:
//     each rank stores its value into slot[parity][my_rank] of EVERY rank's mailbox (plain stores over
//     NVLink), fences, and publishes flag[parity][my_rank] = epoch with a system-scope release store;
//     then it waits (acquire loads) until its own mailbox holds flags >= epoch from all ranks and folds the
//     nranks values in rank order -- the same order on every rank, so all ranks get bit-identical results.
// The epoch lives in the mailbox and is advanced by the kernel itself, so a captured CUDA graph can be
// replayed.  Slots are double-buffered by epoch parity: a rank can only be one all-reduce ahead of the
// slowest rank (finishing epoch e needs everybody's contribution to e), so parity e+2 never overwrites
// values somebody still has to read.
//
// This is what the last block of a reduction kernel runs (block_finish below), which makes "reduce the slice + combine
// across GPUs" ONE kernel with no NCCL call and no host involvement; it replaces the host fold of
// vexcl/reductor.hpp:412-436.
struct PeerArgs {
    unsigned long long *mbox[VEXB_MAX_PEERS];   // mbox[p]: rank p's mailbox as seen from this rank
    int rank, nranks;                           // nranks == 0: disabled
    unsigned long long *fault_host;             // process-wide sticky fault word (mapped pinned host memory), may be NULL
};

// mailbox layout in 8-byte words: [0] epoch, [1] error flag, [16 + ((parity*nranks + src) * 4) + {0,1,2}] = value0, value1, flag
__device__ __forceinline__ unsigned long long *peer_slot(unsigned long long *mbox, int parity, int nranks, int src) {
    return mbox + 16 + (unsigned long long)(parity * nranks + src) * 4;
}

__device__ __forceinline__ void st_release_sys(unsigned long long *p, unsigned long long v) {
    asm volatile("st.release.sys.global.u64 [%0], %1;" :: "l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long ld_acquire_sys(const unsigned long long *p) {
    unsigned long long v;
    asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ unsigned long long ld_relaxed_sys(const unsigned long long *p) {
    unsigned long long v;
    asm volatile("ld.relaxed.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}

// Called by ALL threads of one block (blockDim.x >= nranks).  v0/v1: this rank's contribution as raw 64-bit
// words (thread 0's arguments are used).  On return out0[s]/out1[s] (shared memory, s < nranks) hold every
// rank's words; the caller folds them in rank order.  Returns false (to every thread) when a peer did not arrive
// within ~20 s: the slots are then NOT valid and the caller must not fold them -- it stores NaN / the all-ones
// pattern instead and the fault is made sticky (mailbox word 1 and the process-wide fault word, vexb_peer_fault),
// so that vexb_reduce_fetch and the front ends fail loudly instead of returning a wrong sum.
__device__ __forceinline__ bool peer_exchange(const PeerArgs &pa, unsigned long long v0, unsigned long long v1,
                                              unsigned long long *out0, unsigned long long *out1) {
    __shared__ unsigned long long sh[3];
    __shared__ int sh_ok;
    unsigned long long *mine = pa.mbox[pa.rank];
    if (threadIdx.x == 0) {
        const unsigned long long e = mine[0] + 1;
        mine[0] = e;
        sh[0] = e; sh[1] = v0; sh[2] = v1; sh_ok = 1;
    }
    __syncthreads();
    const unsigned long long e = sh[0];
    const int parity = (int)(e & 1ull);
    if ((int)threadIdx.x < pa.nranks) {
        // push my contribution into rank `threadIdx.x`'s mailbox
        unsigned long long *dst = peer_slot(pa.mbox[threadIdx.x], parity, pa.nranks, pa.rank);
        dst[0] = sh[1]; dst[1] = sh[2];
        __threadfence_system();
        st_release_sys(dst + 2, e);
        // collect rank `threadIdx.x`'s contribution from my own mailbox
        const unsigned long long *src = peer_slot(mine, parity, pa.nranks, threadIdx.x);
        bool ok = ld_acquire_sys(src + 2) >= e;
        if (!ok) {
            unsigned long long t0; asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t0));
            for (unsigned it = 0; !ok; ++it) {
                ok = ld_acquire_sys(src + 2) >= e;
                if (ok) break;
                __nanosleep(it < 64 ? 20 : 200);
                if ((it & 1023u) == 1023u) {
                    unsigned long long t1; asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t1));
                    if (t1 - t0 > 20000000000ull) break;
                }
            }
        }
        if (!ok) {                                  // peer never arrived: sticky fault, nothing is folded
            mine[1] = e;
            if (pa.fault_host) *pa.fault_host = e;
            atomicExch(&sh_ok, 0);
        }
        out0[threadIdx.x] = ok ? ld_relaxed_sys(src) : 0ull;
        out1[threadIdx.x] = ok ? ld_relaxed_sys(src + 1) : 0ull;
    }
    __syncthreads();
    return sh_ok != 0;
}

// What a result holds after a failed exchange: NaN for floating types, all ones for integers.
template <class T> __device__ __forceinline__ T peer_poison() { T v; memset(&v, 0xff, sizeof(T)); return v; }

// Warp shuffle tree -> one partial per block -> the last block to finish (atomic ticket) folds the partials in a fixed
// order -> with a peer group, the combine across GPUs -> result[0] (and result[1] for MINMAX).
template <int OP, class T>
__device__ __forceinline__ void block_finish(Fold<OP, T> f, void *ws, T *result, const PeerArgs &pa) {
    __shared__ T sx[8], sy[8];
    __shared__ bool is_last;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) f.merge(shfl_down_fold<OP, T>(f, off));
    if (lane == 0) { sx[warp] = f.x; sy[warp] = f.y; }
    __syncthreads();
    T *partials = reinterpret_cast<T *>(reinterpret_cast<char *>(ws) + sizeof(ReduceWs));
    unsigned int *ticket = &reinterpret_cast<ReduceWs *>(ws)->ticket;
    if (threadIdx.x == 0) {
        Fold<OP, T> b; b.x = sx[0]; b.y = sy[0];
        for (int w = 1; w < (int)(blockDim.x >> 5); ++w) { Fold<OP, T> o; o.x = sx[w]; o.y = sy[w]; b.merge(o); }
        partials[2 * blockIdx.x] = b.x; partials[2 * blockIdx.x + 1] = b.y;
        __threadfence();
        const unsigned int t = atomicAdd(ticket, 1u);
        is_last = (t == gridDim.x - 1);
    }
    __syncthreads();
    if (!is_last) return;
    __threadfence();
    // last block: fold partials[0..gridDim.x) in a fixed order
    Fold<OP, T> g; g.init();
    if (OP == VEXB_SUM_KAHAN) { /* plain adds from here on */ }
    for (unsigned int b = threadIdx.x; b < gridDim.x; b += blockDim.x) {
        Fold<OP, T> o;
        o.x = __ldcg(&partials[2 * b]); o.y = __ldcg(&partials[2 * b + 1]);
        g.merge(o);
    }
    if (OP == VEXB_SUM_KAHAN) g.y = T(0);
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) g.merge(shfl_down_fold<OP, T>(g, off));
    __syncthreads();
    if (lane == 0) { sx[warp] = g.x; sy[warp] = g.y; }
    __syncthreads();
    if (threadIdx.x == 0) {
        Fold<OP, T> b; b.x = sx[0]; b.y = sy[0];
        for (int w = 1; w < (int)(blockDim.x >> 5); ++w) { Fold<OP, T> o; o.x = sx[w]; o.y = sy[w]; b.merge(o); }
        sx[0] = b.x; sy[0] = b.y;
        *ticket = 0;
    }
    __syncthreads();
    if (pa.nranks > 1) {
        // combine across GPUs in the same kernel: one-hop exchange over NVLink peer memory (peer_exchange above)
        __shared__ unsigned long long px[VEXB_MAX_PEERS], py[VEXB_MAX_PEERS];
        const bool arrived = peer_exchange(pa, to_bits<T>(sx[0]), to_bits<T>(sy[0]), px, py);
        if (threadIdx.x == 0) {
            if (arrived) {
                Fold<OP, T> b; b.x = from_bits<T>(px[0]); b.y = from_bits<T>(py[0]);
                for (int r = 1; r < pa.nranks; ++r) { Fold<OP, T> o; o.x = from_bits<T>(px[r]); o.y = from_bits<T>(py[r]); b.merge(o); }
                sx[0] = b.x; sy[0] = b.y;
            } else { sx[0] = peer_poison<T>(); sy[0] = peer_poison<T>(); }   // a peer timed out: never a partial fold
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        result[0] = sx[0];
        if (OP == VEXB_MINMAX) result[1] = sy[0];
    }
}

} // namespace vexb
#endif
