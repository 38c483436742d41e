#ifndef VEXCL_REDUCTOR_HPP
#define VEXCL_REDUCTOR_HPP
/*
 * vex::Reductor<T, RDC> (vexcl/reductor.hpp:289-439).  The reference reduces each slice to 8*SM
 * partials, copies them to the host and folds them there (:412-436).  Here each device leaves ONE
 * value in device memory (vexb_reduce_all: warp-shuffle fold, last block combines); with several
 * distinct devices the last blocks also exchange their values through peer memory over NVLink
 * inside the same kernel (ncclAllReduce if peer access is unavailable), and one 8-byte copy
 * brings the result back.  When the slices share a device (the reference's own single-GPU test
 * trick) or NCCL is unavailable, the nparts values are folded on the host in device order.
 */
#include <array>
#include <limits>
#include <map>
#include <memory>
#include <mutex>
#include "vector.hpp"

namespace vex {

struct SUM        { static const int op = VEXB_SUM; };
struct SUM_Kahan  { static const int op = VEXB_SUM_KAHAN; };
struct MAX        { static const int op = VEXB_MAX; };
struct MIN        { static const int op = VEXB_MIN; };
/// Combines several reduce operations over one expression (reductor.hpp:132-280): the expression is evaluated once per
/// element and folded by every R (vexb_reduce_multi: one pass over memory).  Result: a CL-style vector with s[k] = R_k.
template <class... R>
struct CombineReductors {
    static_assert(sizeof...(R) >= 1 && sizeof...(R) <= VEXB_MAX_COMBINED, "between 1 and 16 reductors can be combined");
    static const int op = -1;
    static const unsigned count = sizeof...(R);
    static const int *ops() { static const int o[] = { R::op... }; return o; }
};
/// Combined MIN and MAX operation (reductor.hpp:277): the two-value kernel of vexb_reduce_all.
typedef CombineReductors<MIN, MAX> MIN_MAX;

namespace detail {

/// NCCL communicators for a queue list, created on first use; empty when not applicable.
struct comm_set {
    std::vector<vexb_comm*> comms;
    ~comm_set() { for (auto c : comms) vexb_comm_destroy(c); }
};
inline std::shared_ptr<comm_set> communicators(const std::vector<backend::command_queue> &queue) {
    static std::mutex mx;
    static std::map<std::vector<int>, std::shared_ptr<comm_set>> cache;
    std::vector<int> devs;
    for (auto &q : queue) devs.push_back(q.ordinal());
    std::lock_guard<std::mutex> lock(mx);
    auto it = cache.find(devs);
    if (it != cache.end()) return it->second;
    auto cs = std::make_shared<comm_set>();
    std::vector<int> sorted(devs);
    std::sort(sorted.begin(), sorted.end());
    const bool distinct = std::adjacent_find(sorted.begin(), sorted.end()) == sorted.end();
    if (devs.size() > 1 && distinct && !std::getenv("VEXCL_NO_NCCL")) {
        cs->comms.resize(devs.size(), nullptr);
        if (vexb_comm_create_all(static_cast<int>(devs.size()), devs.data(), cs->comms.data()) != VEXB_OK) cs->comms.clear();
    }
    cache[devs] = cs;
    return cs;
}

/// Peer-memory groups (mailboxes mapped between the devices) for a queue list; empty when not applicable.
struct peer_set {
    std::vector<vexb_peer*> peers;
    ~peer_set() { for (auto p : peers) vexb_peer_destroy(p); }
};
inline std::shared_ptr<peer_set> peer_group(const std::vector<backend::command_queue> &queue) {
    static std::mutex mx;
    static std::map<std::vector<int>, std::shared_ptr<peer_set>> cache;
    std::vector<int> devs;
    for (auto &q : queue) devs.push_back(q.ordinal());
    std::lock_guard<std::mutex> lock(mx);
    auto it = cache.find(devs);
    if (it != cache.end()) return it->second;
    auto ps = std::make_shared<peer_set>();
    std::vector<int> sorted(devs);
    std::sort(sorted.begin(), sorted.end());
    const bool distinct = std::adjacent_find(sorted.begin(), sorted.end()) == sorted.end();
    if (devs.size() > 1 && devs.size() <= 16 && distinct && !std::getenv("VEXCL_NO_PEER")) {
        ps->peers.resize(devs.size(), nullptr);
        if (vexb_peer_create_all(static_cast<int>(devs.size()), devs.data(), ps->peers.data()) != VEXB_OK) ps->peers.clear();
    }
    cache[devs] = ps;
    return ps;
}

template <class T, class RDC> struct reduce_result { typedef T type; static const unsigned count = 1; static T make(const T *v) { return v[0]; } };
template <class T, class... R> struct reduce_result<T, CombineReductors<R...>> {
    static const unsigned count = sizeof...(R);
    typedef vecn<T, cl_fit_vec_size<sizeof...(R)>::value> type;
    static type make(const T *v) { type r = type(); for (unsigned k = 0; k < count; ++k) r.s[k] = v[k]; return r; }
};
template <class RDC> struct is_min_max : std::false_type {};
template <> struct is_min_max<CombineReductors<MIN, MAX>> : std::true_type {};

template <class T> inline T host_fold(int op, T a, T b) {
    switch (op) { case VEXB_MAX: return a > b ? a : b; case VEXB_MIN: return a < b ? a : b; default: return a + b; }
}

} // namespace detail

template <typename ScalarType, class RDC = SUM>
class Reductor {
    public:
        typedef typename detail::reduce_result<ScalarType, RDC>::type result_type;

        Reductor(const std::vector<backend::command_queue> &queue
#ifndef VEXCL_NO_STATIC_CONTEXT_CONSTRUCTORS
                = current_context().queue()
#endif
                ) : queue(queue), ws(queue.size()), res(queue.size())
        {
            for (unsigned d = 0; d < queue.size(); ++d) {
                size_t bytes = 0;
                VEXB_CHECKED(vexb_reduce_workspace_bytes(queue[d].ordinal(), &bytes));
                bytes *= detail::reduce_result<ScalarType, RDC>::count;       // combined reductions: one workspace slice each
                ws[d] = backend::device_vector<char>(queue[d], bytes);
                VEXB_CHECKED(vexb_memset(queue[d].ordinal(), ws[d].raw(), 0, bytes, queue[d].raw()));
                res[d] = backend::device_vector<ScalarType>(queue[d], 16);
            }
        }

        template <class Expr>
        typename std::enable_if<is_vector_expr<Expr>::value && detail::ncomp<Expr>::value == 0, result_type>::type
        operator()(const Expr &expr) const { return reduce(detail::operand<Expr>::wrap(expr), -1); }

        /// Multi-expressions reduce component by component (reductor.hpp:341-349).
        template <class Expr>
        typename std::enable_if<is_vector_expr<Expr>::value && (detail::ncomp<Expr>::value > 0),
                                std::array<result_type, detail::ncomp<Expr>::value> >::type
        operator()(const Expr &expr) const {
            std::array<result_type, detail::ncomp<Expr>::value> r;
            for (size_t i = 0; i < r.size(); ++i) r[i] = reduce(expr, static_cast<int>(i));
            return r;
        }
    private:
        template <class Expr>
        result_type reduce(const Expr &expr, int comp) const {
            detail::expr_props p;
            p.comp = comp;
            expr.props(p);
            const int dt = dtype_of<ScalarType>::value;
            const bool combined = RDC::op < 0 && !detail::is_min_max<RDC>::value;
            const int op = detail::is_min_max<RDC>::value ? VEXB_MINMAX : RDC::op;
            const int cnt = static_cast<int>(detail::reduce_result<ScalarType, RDC>::count);
            ScalarType out[16];
            for (int k = 0; k < cnt; ++k) out[k] = identity(op_of(k));
            if (!p.sized || p.size == 0) return detail::reduce_result<ScalarType, RDC>::make(out);   // reductor.hpp:318-321
            if (p.part.empty()) p.part = vex::partition(p.size, queue);                                // :323-325

            // distinct devices: the combine across GPUs happens inside the reduction kernel (peer memory)
            auto ps = queue.size() > 1 ? detail::peer_group(queue) : std::shared_ptr<detail::peer_set>();
            const bool fused = ps && !ps->peers.empty();
            for (unsigned d = 0; d < queue.size(); ++d) {
                detail::ir_builder b(d, comp);
                expr.lower(b);
                const int st = combined
                    ? vexb_reduce_multi(queue[d].ordinal(), queue[d].raw(), &b.e, dt, p.part_size(d), p.part_start(d), cnt, ops_of(),
                                        res[d].raw(), ws[d].raw(), fused ? ps->peers[d] : nullptr)
                    : vexb_reduce_all(queue[d].ordinal(), queue[d].raw(), &b.e, dt, p.part_size(d), p.part_start(d),
                                      op, res[d].raw(), ws[d].raw(), fused ? ps->peers[d] : nullptr);
                if (st == VEXB_ERR_UNSUPPORTED && d == 0) {
                    // NVRTC cannot be loaded, so the kernel that folds user functions and inlined sparse products in one pass
                    // cannot be built: evaluate the expression into a temporary, reduce that
                    vex::vector<typename Expr::value_type> tmp(queue, p.size);
                    detail::assign_expression<assign::SET>(tmp, expr, comp);
                    return reduce(tmp, -1);
                }
                if (st != VEXB_OK && fused && d > 0) {
                    // devices 0..d-1 have already launched and will wait for everybody in the kernel: keep the group in step
                    // (identity + the standalone combine on the devices that did not launch), then report the failure
                    const std::string why = vexb_last_error();
                    for (unsigned e = d; e < queue.size(); ++e)
                        for (int k = 0; k < (combined ? cnt : 1); ++k) {
                            ScalarType *rk = res[e].raw_ptr() + k;
                            vexb_reduce_identity(queue[e].ordinal(), queue[e].raw(), dt, combined ? op_of(k) : op, rk);
                            vexb_peer_allreduce(ps->peers[e], queue[e].raw(), rk, dt, combined ? op_of(k) : op);
                        }
                    throw backend::error(st, why);
                }
                VEXB_CHECKED(st);
            }
            auto cs = (queue.size() > 1 && !fused) ? detail::communicators(queue) : std::shared_ptr<detail::comm_set>();
            if (fused) {
                VEXB_CHECKED(vexb_reduce_fetch(queue[0].ordinal(), queue[0].raw(), res[0].raw(), dt, cnt, out));
            } else if (cs && !cs->comms.empty()) {
                std::vector<void*> bufs, streams;
                for (unsigned d = 0; d < queue.size(); ++d) { bufs.push_back(res[d].raw()); streams.push_back(queue[d].raw()); }
                if (combined) {
                    for (int k = 0; k < cnt; ++k) {
                        std::vector<void*> bk;
                        for (unsigned d = 0; d < queue.size(); ++d) bk.push_back(res[d].raw_ptr() + k);
                        VEXB_CHECKED(vexb_comm_allreduce(static_cast<int>(queue.size()), cs->comms.data(), bk.data(), streams.data(), 1, dt, op_of(k)));
                    }
                } else
                VEXB_CHECKED(vexb_comm_allreduce(static_cast<int>(queue.size()), cs->comms.data(), bufs.data(), streams.data(), 1, dt, op));
                VEXB_CHECKED(vexb_reduce_fetch(queue[0].ordinal(), queue[0].raw(), res[0].raw(), dt, cnt, out));
            } else {
                for (unsigned d = 0; d < queue.size(); ++d) {
                    ScalarType v[16];
                    VEXB_CHECKED(vexb_reduce_fetch(queue[d].ordinal(), queue[d].raw(), res[d].raw(), dt, cnt, v));
                    for (int k = 0; k < cnt; ++k) out[k] = detail::host_fold(op_of(k), out[k], v[k]);
                }
            }
            return detail::reduce_result<ScalarType, RDC>::make(out);
        }
        std::vector<backend::command_queue> queue;
        mutable std::vector<backend::device_vector<char>> ws;
        mutable std::vector<backend::device_vector<ScalarType>> res;

        /// The reduction that produces component k of the result.
        template <class R = RDC> static typename std::enable_if<(R::op >= 0), int>::type op_of(int) { return R::op; }
        template <class R = RDC> static typename std::enable_if<(R::op < 0), int>::type op_of(int k) { return R::ops()[k]; }
        template <class R = RDC> static typename std::enable_if<(R::op >= 0), const int*>::type ops_of() { return nullptr; }
        template <class R = RDC> static typename std::enable_if<(R::op < 0), const int*>::type ops_of() { return R::ops(); }

        static ScalarType identity(int op) {                     // reductor.hpp:55, :87, :111
            switch (op) {
                case VEXB_MAX: return std::numeric_limits<ScalarType>::lowest();
                case VEXB_MIN: return std::numeric_limits<ScalarType>::max();
                default: return ScalarType();
            }
        }
};

template <typename T, class R>
Reductor<T, R> get_reductor(const std::vector<backend::command_queue> &queue) { return Reductor<T, R>(queue); }

} // namespace vex
#endif
