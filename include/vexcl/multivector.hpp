#ifndef VEXCL_MULTIVECTOR_HPP
#define VEXCL_MULTIVECTOR_HPP
/*
 * vex::multivector<T, N> and vex::tie (vexcl/multivector.hpp:121-508, vexcl/operations.hpp:2230-2270):
 * N equally sized vex::vectors that take part in expressions component by component.
 *
 * The reference fuses the N component assignments into one generated kernel.  Here every component
 * is one launch of the same pre-compiled kernels a vex::vector assignment uses (the expression IR is
 * lowered once per component; ir_builder::comp selects the component of every multi-valued terminal).
 * The observable semantics of the fused kernel are kept: all right-hand sides are evaluated before
 * any left-hand side is written -- when a later component reads a vector an earlier one writes, the
 * results go through temporaries (assign_components below).
 *
 * Differences: multivector<T,N>::value_type is T (the reference's sub_value_type); the per-element type
 * std::array<T,N> is multivector<T,N>::element_type.
 */
#include <array>
#include <tuple>
#include <utility>
#include "vector.hpp"

namespace vex {

template <class T, size_t N> class multivector;

namespace detail {

template <class F, size_t... I>
void for_each_index(F &&f, std::index_sequence<I...>) { int dummy[] = {0, (f(std::integral_constant<size_t, I>()), 0)...}; (void)dummy; }

template <class... A> struct all_arithmetic : std::true_type {};
template <class A, class... B> struct all_arithmetic<A, B...>
    : std::integral_constant<bool, std::is_arithmetic<typename std::decay<A>::type>::value && all_arithmetic<B...>::value> {};

/// One scalar per component: std::make_tuple(1, 2, 3, 4) * y, x = std::array<double,4>{...}.
template <class P, size_t N>
struct multi_scalar : vector_expr_tag {
    static const bool hold_by_reference = false;
    static const size_t multi_size = N;
    typedef typename promoted<P>::type value_type;
    std::array<P, N> v;
    int lower(ir_builder &b) const {
        precondition(b.comp >= 0 && static_cast<size_t>(b.comp) < N, "per-component scalars used outside a multi-expression");
        b.push_scalar(v[b.comp]);
        return dtype_of<value_type>::value;
    }
    void props(expr_props&) const {}
};

template <class... A>
struct operand<std::tuple<A...>, void> {
    typedef typename std::common_type<typename std::decay<A>::type...>::type P;
    typedef multi_scalar<P, sizeof...(A)> type;
    static type wrap(const std::tuple<A...> &t) { type r; fill(r, t, std::index_sequence_for<A...>()); return r; }
    private:
        template <size_t... I> static void fill(type &r, const std::tuple<A...> &t, std::index_sequence<I...>) {
            int dummy[] = {0, (r.v[I] = static_cast<P>(std::get<I>(t)), 0)...}; (void)dummy;
        }
};
template <class A, size_t N>
struct operand<std::array<A, N>, void> {
    typedef multi_scalar<A, N> type;
    static type wrap(const std::array<A, N> &a) { type r; r.v = a; return r; }
};
template <class... A> struct is_operand<std::tuple<A...>> : all_arithmetic<A...> {};
template <class A, size_t N> struct is_operand<std::array<A, N>> : std::is_arithmetic<A> {};

/// The same expression for every component (ir_builder::comp picks the component of its multi-valued terminals).
template <class E>
struct same_for_all {
    const E &e;
    template <size_t I> void props(expr_props &p) const { e.props(p); }
    template <size_t I> void lower(ir_builder &b) const { e.lower(b); }
};
/// One expression per component: std::tie(e0, e1, ...) / std::make_tuple(e0, e1, ...).
template <class Tuple>
struct one_per_component {
    const Tuple &t;
    template <size_t I> struct elem { typedef operand<typename std::decay<typename std::tuple_element<I, Tuple>::type>::type> op; };
    template <size_t I> void props(expr_props &p) const { elem<I>::op::wrap(std::get<I>(t)).props(p); }
    template <size_t I> void lower(ir_builder &b) const { elem<I>::op::wrap(std::get<I>(t)).lower(b); }
};

/// lhs[i] OP= component i of the right-hand side, for all i, with the read-everything-then-write semantics of the
/// reference's fused kernel (assign_multiexpression, operations.hpp:2071-2190).
template <class OP, class T, size_t N, class Rhs>
void assign_components(const std::array<vex::vector<T>*, N> &lhs, const Rhs &rhs) {
    const std::vector<backend::command_queue> &queue = lhs[0]->queue_list();
    const size_t nd = queue.size();
    std::vector<ir_builder> ir;                                       // [component][device]
    ir.reserve(N * nd);
    for_each_index([&](auto I) {
        expr_props p;
        constexpr size_t C = decltype(I)::value;
        p.comp = static_cast<int>(C);
        p.see(lhs[C]->queue_list(), lhs[C]->partition(), lhs[C]->size());
        rhs.template props<C>(p);
        for (unsigned d = 0; d < nd; ++d) {
            ir.emplace_back(d, static_cast<int>(C));
            rhs.template lower<C>(ir.back());
        }
    }, std::make_index_sequence<N>());

    // One generated kernel for all components (vexb_eval_multi): reads of element i all happen before its writes, so no
    // temporaries whatever reads what.  Served once the kernel for this tuple of expressions exists (it is compiled in
    // the background at first use); until then -- and for anything it does not take -- component by component below.
    std::vector<backend::device_vector<T>> copies(N * nd);          // [device][target]: what raw pointers into a target read
    {
        bool fused = N >= 2 && N <= 8;
        for (unsigned d = 0; d < nd && fused; ++d) {
            const void *es[N]; void *out[N];
            for (size_t i = 0; i < N; ++i) { es[i] = &ir[i * nd + d].e; out[i] = (*lhs[i])(d).raw(); }
            int handled = 0;
            int st = vexb_eval_multi(queue[d].ordinal(), queue[d].raw(), (int)N, out, dtype_of<T>::value, OP::op,
                                     reinterpret_cast<const vexb_expr *const *>(es), lhs[0]->part_size(d), lhs[0]->part_start(d), &handled);
            // raw pointers into a target read a device copy of it instead (never component by component: that would race
            // too); the component-by-component path below stages through temporaries, so it reads the old targets as is
            bool redirected = false;
            if (st == VEXB_ERR_UNSUPPORTED)
                for (size_t j = 0; j < N; ++j)
                    for (size_t i = 0; i < N; ++i)
                        redirected = redirect_pointers(ir[i * nd + d].e, out[j], dtype_of<T>::value, lhs[j]->part_size(d) * sizeof(T), queue[d],
                                                       copies[d * N + j]) || redirected;
            if (redirected)
                st = vexb_eval_multi(queue[d].ordinal(), queue[d].raw(), (int)N, out, dtype_of<T>::value, OP::op,
                                     reinterpret_cast<const vexb_expr *const *>(es), lhs[0]->part_size(d), lhs[0]->part_start(d), &handled);
            VEXB_CHECKED(st);
            if (!handled) {
                // all devices or none: a kernel that is ready is ready for every device, so only d == 0 can say no
                fused = false;
            }
        }
        if (fused) return;
    }

    bool hazard = false;                                              // does component j > i read what component i writes?
    for (size_t i = 0; i < N && !hazard; ++i)
        for (size_t j = i + 1; j < N && !hazard; ++j)
            for (unsigned d = 0; d < nd && !hazard; ++d) {
                const vexb_expr &e = ir[j * nd + d].e;
                for (int k = 0; k < e.n_terms; ++k)
                    if (e.term[k].kind == VEXB_TERM_VEC && e.term[k].v.ptr == (*lhs[i])(d).raw() && lhs[i]->part_size(d)) hazard = true;
            }

    std::vector<vex::vector<T>> tmp;
    if (hazard) for (size_t i = 0; i + 1 < N; ++i) tmp.emplace_back(queue, lhs[i]->size());   // the last component has no later reader
    for (size_t i = 0; i < N; ++i)
        for (unsigned d = 0; d < nd; ++d) {
            const bool staged = hazard && i + 1 < N;
            VEXB_CHECKED(vexb_eval(queue[d].ordinal(), queue[d].raw(), staged ? tmp[i](d).raw() : (*lhs[i])(d).raw(), dtype_of<T>::value,
                                   staged ? VEXB_SET : OP::op, &ir[i * nd + d].e, lhs[i]->part_size(d), lhs[i]->part_start(d)));
        }
    if (hazard) for (size_t i = 0; i + 1 < N; ++i) assign_expression<OP>(*lhs[i], tmp[i]);
}

/// expression +/- (A * X) for multivectors: evaluated as the expression, then the product appended.
template <class E, class M, class T, size_t N>
struct multi_mixed {
    E expr; additive_operator<M, multivector<T, N>> a;
    multi_mixed(E e, const additive_operator<M, multivector<T, N>> &a) : expr(e), a(a) {}
};

/// Assignment operators shared by multivector (owns its vectors) and vex::tie(...) (refers to vectors).
template <class Derived, class T, size_t N>
struct multi_assignable {
    Derived& self() { return static_cast<Derived&>(*this); }
    std::array<vex::vector<T>*, N> targets() { std::array<vex::vector<T>*, N> t; for (size_t i = 0; i < N; ++i) t[i] = &self()(i); return t; }

#define VEXCL_MULTI_ASSIGNMENT(cop, tag) \
    template <class Expr> \
    typename std::enable_if<is_operand<Expr>::value, const Derived&>::type \
    operator cop(const Expr &expr) { \
        typedef typename operand<Expr>::type held; \
        static_assert(ncomp<held>::value == 0 || ncomp<held>::value == N, "multi-expression has a different number of components"); \
        held h = operand<Expr>::wrap(expr); \
        assign_components<assign::tag>(targets(), same_for_all<typename std::decay<held>::type>{h}); \
        return self(); \
    } \
    template <class... E> \
    typename std::enable_if<!all_arithmetic<E...>::value, const Derived&>::type \
    operator cop(const std::tuple<E...> &t) { \
        static_assert(sizeof...(E) == N, "tuple has a different number of components"); \
        assign_components<assign::tag>(targets(), one_per_component<std::tuple<E...>>{t}); \
        return self(); \
    }
    VEXCL_MULTI_ASSIGNMENT(=, SET) VEXCL_MULTI_ASSIGNMENT(+=, ADD) VEXCL_MULTI_ASSIGNMENT(-=, SUB) VEXCL_MULTI_ASSIGNMENT(*=, MUL)
    VEXCL_MULTI_ASSIGNMENT(/=, DIV) VEXCL_MULTI_ASSIGNMENT(%=, MOD) VEXCL_MULTI_ASSIGNMENT(&=, AND) VEXCL_MULTI_ASSIGNMENT(|=, OR)
    VEXCL_MULTI_ASSIGNMENT(^=, XOR) VEXCL_MULTI_ASSIGNMENT(<<=, LSH) VEXCL_MULTI_ASSIGNMENT(>>=, RSH)
#undef VEXCL_MULTI_ASSIGNMENT

    // Y = A * X and friends (multivector.hpp:395-437)
    template <class M> const Derived& operator=(const additive_operator<M, multivector<T, N>> &a)  { apply(a, T(1), false); return self(); }
    template <class M> const Derived& operator+=(const additive_operator<M, multivector<T, N>> &a) { apply(a, T(1), true);  return self(); }
    template <class M> const Derived& operator-=(const additive_operator<M, multivector<T, N>> &a) { apply(a, T(-1), true); return self(); }
    template <class E, class M> const Derived& operator=(const multi_mixed<E, M, T, N> &m)  { self() = m.expr;  apply(m.a, T(1), true);  return self(); }
    template <class E, class M> const Derived& operator+=(const multi_mixed<E, M, T, N> &m) { self() += m.expr; apply(m.a, T(1), true);  return self(); }
    template <class E, class M> const Derived& operator-=(const multi_mixed<E, M, T, N> &m) { self() -= m.expr; apply(m.a, T(-1), true); return self(); }
    private:
        template <class M> void apply(const additive_operator<M, multivector<T, N>> &a, T sign, bool append) { apply_dispatch(a, sign, append, 0); }
        // an operator that can take all components at once (vex::SpMat: the matrix is streamed once for up to 4 of them) ...
        template <class M>
        auto apply_dispatch(const additive_operator<M, multivector<T, N>> &a, T sign, bool append, int)
            -> decltype(a.A.template apply_multi<N>(a.x, std::declval<Derived&>(), sign, append)) {
            return a.A.template apply_multi<N>(a.x, self(), sign * a.scale, append);
        }
        // ... or one product per component, as the reference does (operations.hpp:876-880)
        template <class M> void apply_dispatch(const additive_operator<M, multivector<T, N>> &a, T sign, bool append, long) {
            for (size_t i = 0; i < N; ++i) a.A.apply(a.x(i), self()(i), sign * a.scale, append);
        }
};

/// vex::tie(a, b, ...) (operations.hpp:2252): assignable group of existing vectors.
template <class T, size_t N>
struct tied_vectors : vector_expr_tag, multi_assignable<tied_vectors<T, N>, T, N> {
    static const bool hold_by_reference = false;
    static const size_t multi_size = N;
    typedef T value_type;
    std::array<vex::vector<T>*, N> v;
    vex::vector<T>& operator()(size_t i) { return *v[i]; }
    const vex::vector<T>& operator()(size_t i) const { return *v[i]; }
    size_t size() const { return v[0]->size(); }
    using multi_assignable<tied_vectors<T, N>, T, N>::operator=;
    const tied_vectors& operator=(const tied_vectors &o) {
        std::array<vex::vector<T>*, N> t = v;
        assign_components<assign::SET>(t, same_for_all<tied_vectors>{o});
        return *this;
    }
    int lower(ir_builder &b) const {
        precondition(b.comp >= 0 && static_cast<size_t>(b.comp) < N, "vex::tie used outside a multi-expression");
        return v[b.comp]->lower(b);
    }
    void props(expr_props &p) const { v[p.comp >= 0 ? p.comp : 0]->props(p); }
};

} // namespace detail

template <class T, size_t N>
class multivector : public vector_expr_tag, public detail::multi_assignable<multivector<T, N>, T, N> {
    public:
        static const bool hold_by_reference = true;
        static const size_t multi_size = N;
        static const size_t NDIM = N;
        typedef T value_type;
        typedef T sub_value_type;
        typedef vex::vector<T> subtype;
        typedef std::array<T, N> element_type;

        /// Proxy for one element of every component (multivector.hpp:127-165).
        class element {
            public:
                operator element_type() const { element_type e; for (size_t i = 0; i < N; ++i) e[i] = (*mv)(i)[index]; return e; }
                element_type operator=(element_type e) { for (size_t i = 0; i < N; ++i) (*mv)(i)[index] = e[i]; return e; }
            private:
                element(multivector &m, size_t i) : mv(&m), index(i) {}
                multivector *mv; size_t index;
                friend class multivector;
        };
        template <class MV>
        struct iterator_type {
            MV *mv; size_t pos;
            iterator_type(MV &m, size_t p) : mv(&m), pos(p) {}
            iterator_type& operator++() { ++pos; return *this; }
            iterator_type operator+(ptrdiff_t d) const { return iterator_type(*mv, pos + d); }
            ptrdiff_t operator-(const iterator_type &o) const { return static_cast<ptrdiff_t>(pos) - static_cast<ptrdiff_t>(o.pos); }
            bool operator==(const iterator_type &o) const { return pos == o.pos; }
            bool operator!=(const iterator_type &o) const { return pos != o.pos; }
            auto operator*() const -> decltype((*mv)[pos]) { return (*mv)[pos]; }
        };
        typedef iterator_type<multivector> iterator;
        typedef iterator_type<const multivector> const_iterator;

        multivector() {}
        /// Host data holds the components one after another (multivector.hpp:232-246).
        multivector(const std::vector<backend::command_queue> &queue, const std::vector<T> &host,
                    backend::mem_flags flags = backend::MEM_READ_WRITE) {
            const size_t size = host.size() / N;
            precondition(N * size == host.size(), "multivector: host data is not a multiple of the component count");
            for (size_t i = 0; i < N; ++i) vex::vector<T>(queue, size, host.data() + i * size, flags).swap(vec[i]);
        }
        multivector(const std::vector<backend::command_queue> &queue, size_t size, const T *host = 0,
                    backend::mem_flags flags = backend::MEM_READ_WRITE) {
            for (size_t i = 0; i < N; ++i) vex::vector<T>(queue, size, host ? host + i * size : 0, flags).swap(vec[i]);
        }
#ifndef VEXCL_NO_STATIC_CONTEXT_CONSTRUCTORS
        explicit multivector(size_t size) { for (size_t i = 0; i < N; ++i) vec[i].resize(size); }
#endif
        multivector(const multivector &mv) : vector_expr_tag(), detail::multi_assignable<multivector, T, N>() {
            for (size_t i = 0; i < N; ++i) vec[i].resize(mv(i));
        }
        multivector(multivector &&mv) noexcept { for (size_t i = 0; i < N; ++i) vec[i].swap(mv.vec[i]); }

        void resize(const std::vector<backend::command_queue> &queue, size_t size) { for (size_t i = 0; i < N; ++i) vec[i].resize(queue, size); }
        void resize(size_t size) { for (size_t i = 0; i < N; ++i) vec[i].resize(size); }
        void clear() { *this = static_cast<T>(0); }
        void swap(multivector &o) { for (size_t i = 0; i < N; ++i) vec[i].swap(o.vec[i]); }

        size_t size() const { return vec[0].size(); }
        const vex::vector<T>& operator()(size_t i) const { return vec[i]; }
        vex::vector<T>& operator()(size_t i) { return vec[i]; }
        const_iterator begin() const { return const_iterator(*this, 0); }
        const_iterator end() const { return const_iterator(*this, size()); }
        iterator begin() { return iterator(*this, 0); }
        iterator end() { return iterator(*this, size()); }
        element_type operator[](size_t i) const { element_type e; for (size_t c = 0; c < N; ++c) e[c] = vec[c][i]; return e; }
        element operator[](size_t i) { return element(*this, i); }
        const std::vector<backend::command_queue>& queue_list() const { return vec[0].queue_list(); }
        const std::vector<size_t>& partition() const { return vec[0].partition(); }

        using detail::multi_assignable<multivector, T, N>::operator=;
        const multivector& operator=(const multivector &mv) {
            if (&mv != this) for (size_t i = 0; i < N; ++i) vec[i] = mv.vec[i];
            return *this;
        }
        const multivector& operator=(multivector &&mv) { swap(mv); return *this; }

        // expression terminal protocol: component ir_builder::comp
        int lower(detail::ir_builder &b) const {
            precondition(b.comp >= 0 && static_cast<size_t>(b.comp) < N, "multivector used in a single-vector expression");
            return vec[b.comp].lower(b);
        }
        void props(detail::expr_props &p) const { vec[0].props(p); }
    private:
        std::array<vex::vector<T>, N> vec;
};

template <class T, size_t N> void swap(multivector<T, N> &x, multivector<T, N> &y) { x.swap(y); }

/// Host <-> device, components one after another (multivector.hpp:510-525).
template <class T, size_t N> void copy(const multivector<T, N> &mv, std::vector<T> &hv) {
    precondition(hv.size() == N * mv.size(), "vex::copy: sizes differ");
    for (size_t i = 0; i < N; ++i) mv(i).read_data(0, mv.size(), hv.data() + i * mv.size(), true);
}
template <class T, size_t N> void copy(const std::vector<T> &hv, multivector<T, N> &mv) {
    precondition(hv.size() == N * mv.size(), "vex::copy: sizes differ");
    for (size_t i = 0; i < N; ++i) mv(i).write_data(0, mv.size(), hv.data() + i * mv.size(), true);
}

/// vex::tie(a, b) = std::tie(a + b, a - b);
template <class T, class... Rest>
detail::tied_vectors<T, 1 + sizeof...(Rest)> tie(vex::vector<T> &first, Rest&... rest) {
    detail::tied_vectors<T, 1 + sizeof...(Rest)> t;
    t.v = {{&first, &rest...}};
    return t;
}

// expression +/- A * X
template <class E, class M, class T, size_t N>
typename std::enable_if<detail::is_operand<E>::value, detail::multi_mixed<typename detail::operand<E>::type, M, T, N> >::type
operator+(const E &e, const additive_operator<M, multivector<T, N>> &a) {
    return detail::multi_mixed<typename detail::operand<E>::type, M, T, N>(detail::operand<E>::wrap(e), a);
}
template <class E, class M, class T, size_t N>
typename std::enable_if<detail::is_operand<E>::value, detail::multi_mixed<typename detail::operand<E>::type, M, T, N> >::type
operator+(const additive_operator<M, multivector<T, N>> &a, const E &e) { return e + a; }
template <class E, class M, class T, size_t N>
typename std::enable_if<detail::is_operand<E>::value, detail::multi_mixed<typename detail::operand<E>::type, M, T, N> >::type
operator-(const E &e, const additive_operator<M, multivector<T, N>> &a) {
    return detail::multi_mixed<typename detail::operand<E>::type, M, T, N>(detail::operand<E>::wrap(e), -a);
}

template <class T, size_t N>
std::ostream& operator<<(std::ostream &o, const multivector<T, N> &t) {
    std::vector<T> h(N * t.size());
    copy(t, h);
    o << "{";
    for (size_t i = 0; i < t.size(); ++i) {
        if (i % 4 == 0) o << "\n" << std::setw(6) << i << ":";
        o << " (";
        for (size_t j = 0; j < N; ++j) o << " " << h[j * t.size() + i];
        o << ")";
    }
    return o << "\n}\n";
}

} // namespace vex
#endif
