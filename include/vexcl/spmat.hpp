#ifndef VEXCL_SPMAT_HPP
#define VEXCL_SPMAT_HPP
/*
 * vex::SpMat<val_t, col_t, idx_t> (vexcl/spmat.hpp:56-386): CSR in, one row strip per device,
 * ghost columns exchanged between devices, `y = A * x`, `y += A * x`, `y -= 2 * (A * x)`, ...
 *
 * What changed behind the same interface:
 *   - strips are stored with 32-bit local indices and multiplied by hand-written sm_90a
 *     kernels (row-block CSR stream with TMA staging, or hybrid ELL; libvexb200 picks);
 *   - the ghost exchange (reference: D2H, host shuffle, H2D with three host syncs,
 *     spmat.hpp:137-175) happens inside the product kernel: it stores the values its neighbours
 *     need straight into their ghost buffers over NVLink peer memory and waits for its own
 *     (one launch per device and product; csrc/distapply.cu).  Without peer access: grouped
 *     ncclSend/ncclRecv on a side stream.  Nothing in apply() waits on the host.
 */
#include <memory>
#include "reductor.hpp"
#include "vector.hpp"
#include "multivector.hpp"

namespace vex {

template <typename val_t, typename col_t = size_t, typename idx_t = size_t>
class SpMat {
    public:
        typedef val_t value_type;
        typedef val_t scalar_type;

        SpMat() : nrows(0), ncols(0), nnz(0), plan(nullptr) {}

        SpMat(const std::vector<backend::command_queue> &queue, size_t n, size_t m,
              const idx_t *row, const col_t *col, const val_t *val, int format = VEXB_FMT_AUTO)
            : queue(queue), part(vex::partition(n, queue)), col_part(vex::partition(m, queue)),
              nrows(n), ncols(m), nnz(row[n]), plan(nullptr), mtx(queue.size(), nullptr)
        {
            static_assert(sizeof(col_t) == 4 || sizeof(col_t) == 8, "column type must be 32 or 64 bit");
            static_assert(sizeof(idx_t) == 4 || sizeof(idx_t) == 8, "index type must be 32 or 64 bit");
            const int nd = static_cast<int>(queue.size());
            // ghost columns of each strip (spmat.hpp:300-316)
            std::vector<int64_t> ghosts; std::vector<size_t> off(nd + 1, 0);
            for (int d = 0; d < nd; ++d) {
                size_t cnt = 0;
                if (nd > 1) {
                    const size_t nloc = part[d + 1] - part[d];
                    VEXB_CHECKED(vexb_strip_ghost_cols(nloc, row + part[d], sizeof(idx_t), col + row[part[d]], sizeof(col_t),
                                                       col_part[d], col_part[d + 1], nullptr, &cnt));
                    ghosts.resize(off[d] + cnt);
                    size_t cap = cnt;
                    VEXB_CHECKED(vexb_strip_ghost_cols(nloc, row + part[d], sizeof(idx_t), col + row[part[d]], sizeof(col_t),
                                                       col_part[d], col_part[d + 1], ghosts.data() + off[d], &cap));
                }
                off[d + 1] = off[d] + cnt;
            }
            VEXB_CHECKED(vexb_halo_plan_create(nd, col_part.data(), ghosts.data(), off.data(), &plan));
            for (int d = 0; d < nd; ++d) {
                const size_t nloc = part[d + 1] - part[d];
                VEXB_CHECKED(vexb_dspmat_create(queue[d].ordinal(), queue[d].raw(), d, plan, nloc, row + part[d], sizeof(idx_t),
                                                col + row[part[d]], sizeof(col_t), val + row[part[d]], dtype_of<val_t>::value,
                                                format, &mtx[d]));
            }
            if (nd > 1 && off[nd] > 0) {
                // distinct devices with peer access: the halo is pushed through NVLink peer memory inside the product kernel
                // (one launch per device and product); otherwise NCCL send/recv or copy-engine copies
                bool distinct = nd <= 16;
                for (int a = 0; distinct && a < nd; ++a) for (int b = a + 1; b < nd; ++b) if (queue[a].ordinal() == queue[b].ordinal()) distinct = false;
                peer_halo = distinct && vexb_dspmat_halo_connect_local(nd, mtx.data()) == VEXB_OK;
                if (distinct && !peer_halo) for (auto m : mtx) vexb_dspmat_halo_disconnect(m);
                if (!peer_halo) comms = detail::communicators(queue);
            }
        }

        SpMat(const SpMat&) = delete;
        SpMat& operator=(const SpMat&) = delete;
        SpMat(SpMat &&o) noexcept : SpMat() { swap(o); }
        SpMat& operator=(SpMat &&o) noexcept { swap(o); return *this; }
        ~SpMat() {
            for (auto m : mtx) vexb_dspmat_destroy(m);
            if (plan) vexb_halo_plan_destroy(plan);
        }

        /// y = alpha * A * x   or   y += alpha * A * x   (spmat.hpp:120-185).
        void apply(const vex::vector<val_t> &x, vex::vector<val_t> &y, scalar_type alpha = 1, bool append = false) const {
            precondition(x.size() == ncols && y.size() == nrows, "SpMat::apply: vector sizes do not match the matrix");
            const int nd = static_cast<int>(queue.size());
            std::vector<const void*> xs(nd); std::vector<void*> ys(nd), streams(nd);
            for (int d = 0; d < nd; ++d) { xs[d] = x(d).raw(); ys[d] = y(d).raw(); streams[d] = queue[d].raw(); }
            vexb_comm *const *cm = (comms && !comms->comms.empty()) ? comms->comms.data() : nullptr;
            VEXB_CHECKED(vexb_dspmat_apply(nd, cm, mtx.data(), streams.data(), xs.data(), ys.data(), static_cast<double>(alpha), append));
        }

        /// Y(i) = alpha * A * X(i) (or +=) for all N components; the matrix is read once per group of up to four components
        /// when the strips have no halo (vexb_dspmat_apply_multi; the reference multiplies component by component).
        template <size_t N, class X, class Y>
        void apply_multi(const X &x, Y &y, scalar_type alpha = 1, bool append = false) const {
            const int nd = static_cast<int>(queue.size());
            std::vector<const void*> xs(nd * N); std::vector<void*> ys(nd * N), streams(nd);
            for (size_t i = 0; i < N; ++i)
                precondition(x(i).size() == ncols && y(i).size() == nrows, "SpMat::apply: vector sizes do not match the matrix");
            for (int d = 0; d < nd; ++d) {
                streams[d] = queue[d].raw();
                for (size_t i = 0; i < N; ++i) { xs[d * N + i] = x(i)(d).raw(); ys[d * N + i] = y(i)(d).raw(); }
            }
            vexb_comm *const *cm = (comms && !comms->comms.empty()) ? comms->comms.data() : nullptr;
            VEXB_CHECKED(vexb_dspmat_apply_multi(nd, cm, mtx.data(), streams.data(), static_cast<int>(N), xs.data(), ys.data(),
                                                 static_cast<double>(alpha), append));
        }

        /// The strip of device d when it can be inlined into an expression kernel (no halo, plain CSR / hybrid ELL), else NULL.
        const vexb_spmat* inline_strip(unsigned d) const {
            const vexb_spmat *s = nullptr;
            if (d < mtx.size() && mtx[d]) vexb_dspmat_inline_strip(mtx[d], &s);
            return s;
        }
        /// The strip of device d when an assignment can take it as a terminal by sweeping in its storage order (no halo,
        /// plain sliced ELL), else NULL.
        const vexb_spmat* sweep_strip(unsigned d) const {
            const vexb_spmat *s = nullptr;
            if (d < mtx.size() && mtx[d]) vexb_dspmat_sweep_strip(mtx[d], &s);
            return s;
        }
        const std::vector<backend::command_queue>& queue_list() const { return queue; }
        bool inlinable() const { for (unsigned d = 0; d < mtx.size(); ++d) if (!inline_strip(d)) return false; return !mtx.empty(); }

        size_t rows() const { return nrows; }
        size_t cols() const { return ncols; }
        size_t nonzeros() const { return nnz; }
        vexb_dspmat_info info(unsigned d = 0) const { vexb_dspmat_info i; VEXB_CHECKED(vexb_dspmat_get_info(mtx[d], &i)); return i; }
    private:
        std::vector<backend::command_queue> queue;
        std::vector<size_t> part, col_part;
        size_t nrows, ncols, nnz;
        vexb_halo_plan *plan;
        std::vector<vexb_dspmat*> mtx;
        std::shared_ptr<detail::comm_set> comms;
        bool peer_halo = false;

        void swap(SpMat &o) {
            std::swap(queue, o.queue); std::swap(part, o.part); std::swap(col_part, o.col_part);
            std::swap(nrows, o.nrows); std::swap(ncols, o.ncols); std::swap(nnz, o.nnz);
            std::swap(plan, o.plan); std::swap(mtx, o.mtx); std::swap(comms, o.comms); std::swap(peer_halo, o.peer_halo);
        }
};

template <typename val_t, typename col_t, typename idx_t>
additive_operator<SpMat<val_t, col_t, idx_t>, vector<val_t>>
operator*(const SpMat<val_t, col_t, idx_t> &A, const vector<val_t> &x) {
    return additive_operator<SpMat<val_t, col_t, idx_t>, vector<val_t>>(A, x);
}

/// `A * x` as a terminal of any vector expression (vexcl/spmat/inline_spmv.hpp:42-76), e.g.
///     eps = sum(fabs(f - vex::make_inline(A * x)));
/// As in the reference, the row loop is generated into the consumer's kernel (VEXB_TERM_SPMV, NVRTC) whenever the
/// strips have no halo (one device, or a block-diagonal matrix); otherwise -- which the reference forbids -- the product is
/// evaluated by the SpMV kernels into a temporary when the enclosing expression is launched.
template <class M, class V>
struct inline_spmv : vector_expr_tag {
    static const bool hold_by_reference = false;
    typedef typename V::value_type value_type;
    const M &A; const V &x;
    mutable std::shared_ptr<vex::vector<value_type>> y;
    inline_spmv(const M &A, const V &x) : A(A), x(x) {}
    void props(detail::expr_props &p) const {
        fused = std::is_floating_point<value_type>::value && x.size() == A.cols() && (A.inlinable() || p.claim_sweep(A));
        if (fused) { p.see(x.queue_list(), vex::partition(A.rows(), x.queue_list()), A.rows()); return; }   // the row loop goes into the consumer's kernel
        if (!y || y->size() != A.rows()) y = std::make_shared<vex::vector<value_type>>(x.queue_list(), A.rows());
        A.apply(x, *y, 1, false);
        y->props(p);
    }
    int lower(detail::ir_builder &b) const {
        if (!fused) return y->lower(b);
        const vexb_spmat *s = A.inline_strip(b.part);
        b.push_spmv(s ? s : A.sweep_strip(b.part), x(b.part).raw(), dtype_of<value_type>::value);
        return dtype_of<value_type>::value;
    }
    mutable bool fused = false;
};

template <typename val_t, typename col_t, typename idx_t>
const inline_spmv<SpMat<val_t, col_t, idx_t>, vector<val_t>>
make_inline(const additive_operator<SpMat<val_t, col_t, idx_t>, vector<val_t>> &base) {
    precondition(base.scale == 1, "make_inline: scale the inlined product inside the expression instead");
    return inline_spmv<SpMat<val_t, col_t, idx_t>, vector<val_t>>(base.A, base.x);
}

// ---- multivectors: one product per component (spmat.hpp:188-196, inline_spmv.hpp:78-106) ----------------------------
template <typename val_t, typename col_t, typename idx_t, size_t N>
additive_operator<SpMat<val_t, col_t, idx_t>, multivector<val_t, N>>
operator*(const SpMat<val_t, col_t, idx_t> &A, const multivector<val_t, N> &x) {
    return additive_operator<SpMat<val_t, col_t, idx_t>, multivector<val_t, N>>(A, x);
}

template <class M, class T, size_t N>
struct inline_multi_spmv : vector_expr_tag {
    static const bool hold_by_reference = false;
    static const size_t multi_size = N;
    typedef T value_type;
    const M &A; const multivector<T, N> &x;
    mutable std::shared_ptr<multivector<T, N>> y;
    inline_multi_spmv(const M &A, const multivector<T, N> &x) : A(A), x(x) {}
    void props(detail::expr_props &p) const {
        precondition(p.comp >= 0 && static_cast<size_t>(p.comp) < N, "inlined multivector product used in a single-vector expression");
        if (!y || y->size() != A.rows()) y = std::make_shared<multivector<T, N>>(x.queue_list(), A.rows());
        A.apply(x(p.comp), (*y)(p.comp), 1, false);
        (*y)(p.comp).props(p);
    }
    int lower(detail::ir_builder &b) const { return y->lower(b); }
};

template <typename val_t, typename col_t, typename idx_t, size_t N>
const inline_multi_spmv<SpMat<val_t, col_t, idx_t>, val_t, N>
make_inline(const additive_operator<SpMat<val_t, col_t, idx_t>, multivector<val_t, N>> &base) {
    precondition(base.scale == 1, "make_inline: scale the inlined product inside the expression instead");
    return inline_multi_spmv<SpMat<val_t, col_t, idx_t>, val_t, N>(base.A, base.x);
}

} // namespace vex
#endif
