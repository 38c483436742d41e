#ifndef VEXCL_VECTOR_HPP
#define VEXCL_VECTOR_HPP
/*
 * vex::vector<T>: a dense vector cut into contiguous slices, one per queue of the context
 * (vexcl/vector.hpp:220-935), with the reference's partitioning rule (:131-167), the
 * assignment family (:666-801) and the copy() helpers (:998-1228).
 *
 * Default partitioning differs on purpose: the reference weighs devices by a timing of
 * `a = b + c` at first use (device_vector_perf, :1237-1255), which makes slice boundaries
 * timing dependent; on a homogeneous multi-GPU H100 node the default here is equal_weights.
 * set_partitioning(device_vector_perf) restores the measured behaviour.
 */
#include <algorithm>
#include <functional>
#include <iostream>
#include <map>
#include <mutex>
#include <vector>
#include "backend.hpp"
#include "devlist.hpp"
#include "operations.hpp"
#include "profiler.hpp"
#include "types.hpp"
#include "util.hpp"

namespace vex {

inline double equal_weights(const backend::command_queue&) { return 1; }
inline double device_vector_perf(const backend::command_queue&);

namespace detail {
struct partitioning_state {
    std::function<double(const backend::command_queue&)> weight = equal_weights;
    bool is_set = false;
    std::map<backend::device_id, double> device_weight;
    std::mutex mx;
    static partitioning_state& get() { static partitioning_state s; return s; }
};
}

/// Set the device weighting function; only the first call takes effect (vector.hpp:94-106).
inline void set_partitioning(std::function<double(const backend::command_queue&)> f) {
    auto &s = detail::partitioning_state::get();
    std::lock_guard<std::mutex> lock(s.mx);
    if (!s.is_set) { s.weight = f; s.is_set = true; }
    else std::cerr << "Warning: device weighting function is already set and will be left as is." << std::endl;
}

/// Slice boundaries of an n-element container over the given queues.
inline std::vector<size_t> partition(size_t n, const std::vector<backend::command_queue> &queue) {
    std::vector<size_t> part(queue.size() + 1, 0);
    if (queue.empty()) return part;
    std::vector<double> w(queue.size(), 1.0);
    if (queue.size() > 1) {
        auto &s = detail::partitioning_state::get();
        std::function<double(const backend::command_queue&)> weight;
        { std::lock_guard<std::mutex> lock(s.mx); weight = s.weight; s.is_set = true; }
        for (size_t d = 0; d < queue.size(); ++d) {
            const backend::device_id id = backend::get_device_id(queue[d]);
            bool known; double val = 1;
            { std::lock_guard<std::mutex> lock(s.mx); auto it = s.device_weight.find(id); known = it != s.device_weight.end(); if (known) val = it->second; }
            if (!known) { val = weight(queue[d]); std::lock_guard<std::mutex> lock(s.mx); s.device_weight[id] = val; }
            w[d] = val;
        }
    }
    VEXB_CHECKED(vexb_partition(n, static_cast<int>(queue.size()), w.data(), part.data()));
    return part;
}

template <typename T>
class vector : public vector_expr_tag {
    public:
        typedef T value_type;
        typedef size_t size_type;
        static const bool hold_by_reference = true;

        /// Proxy for one element: reads and writes are one-element copies (vector.hpp:232-270).
        class element {
            public:
                operator T() const { T v; buf.read(q, index, 1, &v, true); return v; }
                T operator=(T v) { buf.write(q, index, 1, &v, true); return v; }
                T operator=(const element &o) { return *this = static_cast<T>(o); }
            private:
                element(const backend::command_queue &q, const backend::device_vector<T> &b, size_t i) : q(q), buf(b), index(i) {}
                const backend::command_queue &q; backend::device_vector<T> buf; size_t index;
                friend class vector;
        };

        /// Position marker used by copy() (vector.hpp:272-353).
        template <class V>
        struct iterator_type {
            V *vec; size_t pos;
            iterator_type(V &v, size_t p) : vec(&v), pos(p) {}
            iterator_type operator+(ptrdiff_t d) const { return iterator_type(*vec, pos + d); }
            iterator_type& operator++() { ++pos; return *this; }
            iterator_type& operator+=(ptrdiff_t d) { pos += d; return *this; }
            ptrdiff_t operator-(const iterator_type &o) const { return static_cast<ptrdiff_t>(pos) - static_cast<ptrdiff_t>(o.pos); }
            bool operator==(const iterator_type &o) const { return pos == o.pos; }
            bool operator!=(const iterator_type &o) const { return pos != o.pos; }
        };
        typedef iterator_type<vector> iterator;
        typedef iterator_type<const vector> const_iterator;

        vector() {}

        vector(const std::vector<backend::command_queue> &queue, size_t size, const T *host = 0,
               backend::mem_flags flags = backend::MEM_READ_WRITE)
            : queue(queue), part(vex::partition(size, queue)), buf(queue.size())
        { allocate_buffers(flags, host); }

        vector(const std::vector<backend::command_queue> &queue, const std::vector<T> &host,
               backend::mem_flags flags = backend::MEM_READ_WRITE)
            : queue(queue), part(vex::partition(host.size(), queue)), buf(queue.size())
        { allocate_buffers(flags, host.data()); }

        /// Wrap an existing device buffer (single queue).
        vector(const backend::command_queue &q, const backend::device_vector<T> &buffer, size_t size = 0)
            : queue(1, q), part(2), buf(1, buffer)
        { part[0] = 0; part[1] = size ? size : buffer.size(); }

#ifndef VEXCL_NO_STATIC_CONTEXT_CONSTRUCTORS
        explicit vector(size_t size) : vector(current_context().queue(), size) {}
        explicit vector(const std::vector<T> &host) : vector(current_context().queue(), host) {}
#endif

        vector(const vector &v) : vector_expr_tag(), queue(v.queue), part(v.part), buf(v.queue.size()) {
            allocate_buffers(backend::MEM_READ_WRITE, 0);
            *this = v;
        }
        vector(vector &&v) noexcept { swap(v); }

        /// Construct from an expression; size and queues come from its first vector terminal.
        template <class Expr, class = typename std::enable_if<is_vector_expr<Expr>::value && !std::is_same<typename std::decay<Expr>::type, vector>::value>::type>
        vector(const Expr &expr) {
            detail::expr_props p;
            expr.props(p);
            precondition(p.queue && p.sized, "Can not determine expression size and queue list");
            queue = *p.queue; part = p.part.empty() ? vex::partition(p.size, queue) : p.part; buf.resize(queue.size());
            allocate_buffers(backend::MEM_READ_WRITE, 0);
            *this = expr;
        }

        void swap(vector &v) { std::swap(queue, v.queue); std::swap(part, v.part); std::swap(buf, v.buf); }
        void resize(const vector &v) { vector(v).swap(*this); }
        void resize(const std::vector<backend::command_queue> &q, size_t size, const T *host = 0) { vector(q, size, host).swap(*this); }
        void resize(const std::vector<backend::command_queue> &q, const std::vector<T> &host) { vector(q, host).swap(*this); }
        void resize(size_t size) { vector(queue.empty() ? current_context().queue() : queue, size).swap(*this); }
        void clear() { *this = static_cast<T>(0); }

        const backend::device_vector<T>& operator()(unsigned d = 0) const { return buf[d]; }
        backend::device_vector<T>& operator()(unsigned d = 0) { return buf[d]; }

        const_iterator begin() const { return const_iterator(*this, 0); }
        const_iterator end() const { return const_iterator(*this, size()); }
        iterator begin() { return iterator(*this, 0); }
        iterator end() { return iterator(*this, size()); }

        const element operator[](size_t index) const {
            size_t d = std::upper_bound(part.begin(), part.end(), index) - part.begin() - 1;
            return element(queue[d], buf[d], index - part[d]);
        }
        element operator[](size_t index) {
            size_t d = std::upper_bound(part.begin(), part.end(), index) - part.begin() - 1;
            return element(queue[d], buf[d], index - part[d]);
        }
        const element at(size_t index) const { if (index >= size()) throw std::out_of_range("vex::vector"); return (*this)[index]; }
        element at(size_t index) { if (index >= size()) throw std::out_of_range("vex::vector"); return (*this)[index]; }

        size_t size() const { return part.empty() ? 0 : part.back(); }
        size_t nparts() const { return queue.size(); }
        size_t part_size(unsigned d) const { return part[d + 1] - part[d]; }
        size_t part_start(unsigned d) const { return part[d]; }
        const std::vector<backend::command_queue>& queue_list() const { return queue; }
        const std::vector<size_t>& partition() const { return part; }

        typename backend::device_vector<T>::mapped_array map(unsigned d = 0) { return buf[d].map(queue[d]); }
        typename backend::device_vector<T>::mapped_array map(unsigned d = 0) const { return buf[d].map(queue[d]); }

        // ---- assignment family (vector.hpp:666-801) -----------------------------------------
        const vector& operator=(const vector &x) {
            if (&x != this) detail::assign_expression<assign::SET>(*this, x);
            return *this;
        }
        const vector& operator=(vector &&v) { swap(v); return *this; }

#define VEXCL_ASSIGNMENT(cop, tag) \
        template <class Expr> \
        typename std::enable_if<detail::is_operand<Expr>::value, const vector&>::type \
        operator cop(const Expr &expr) { \
            static_assert(detail::ncomp<typename detail::operand<Expr>::type>::value == 0, \
                          "a multi-expression can only be assigned to a multivector or vex::tie(...)"); \
            detail::assign_expression<assign::tag>(*this, detail::operand<Expr>::wrap(expr)); \
            return *this; \
        }
        VEXCL_ASSIGNMENT(=, SET) VEXCL_ASSIGNMENT(+=, ADD) VEXCL_ASSIGNMENT(-=, SUB) VEXCL_ASSIGNMENT(*=, MUL)
        VEXCL_ASSIGNMENT(/=, DIV) VEXCL_ASSIGNMENT(%=, MOD) VEXCL_ASSIGNMENT(&=, AND) VEXCL_ASSIGNMENT(|=, OR)
        VEXCL_ASSIGNMENT(^=, XOR) VEXCL_ASSIGNMENT(<<=, LSH) VEXCL_ASSIGNMENT(>>=, RSH)
#undef VEXCL_ASSIGNMENT

        // additive operators: y = A*x, y += A*x, y -= A*x, and sums of them (vector.hpp:698-801)
        template <class M> const vector& operator=(const additive_operator<M, vector> &a)  { a.apply(*this, T(1), false); return *this; }
        template <class M> const vector& operator+=(const additive_operator<M, vector> &a) { a.apply(*this, T(1), true);  return *this; }
        template <class M> const vector& operator-=(const additive_operator<M, vector> &a) { a.apply(*this, T(-1), true); return *this; }
        // block sparse products (sparse/matrix.hpp): one launch straight into y
        template <class M> const vector& operator=(const direct_product<M, vector> &p)  { p.A.mul(p.x, *this, 1, false); return *this; }
        template <class M> const vector& operator+=(const direct_product<M, vector> &p) { p.A.mul(p.x, *this, 1, true);  return *this; }
        template <class M> const vector& operator-=(const direct_product<M, vector> &p) {
            static_assert(detail::direct_scales<M>::value, "a product of a matrix of user value types is not negated: its "
                          "spmv_ops_impl has no hook for it, so only Y = A * X and Y += A * X are defined");
            p.A.mul(p.x, *this, -1, true); return *this;
        }
        const vector& operator=(const detail::additive_terms<T> &a)  { apply_terms(a, T(1), false); return *this; }
        const vector& operator+=(const detail::additive_terms<T> &a) { apply_terms(a, T(1), true);  return *this; }
        const vector& operator-=(const detail::additive_terms<T> &a) { apply_terms(a, T(-1), true); return *this; }
        // vector part first, then each additive term appended (vector.hpp:758-763)
        // When every product can be inlined (strips without a halo) the whole right-hand side is ONE generated kernel:
        // `y = x + A*x` reads A and x once and writes y once (sparse/product.hpp:45-130 is the reference's fused form).
        template <class E> const vector& operator=(const mixed_expression<E, T> &m) {
            if (inlinable(m.terms)) { detail::assign_expression<assign::SET>(*this, detail::fused_mixed<E, T>(m.expr, m.terms, T(1))); return *this; }
            *this = m.expr;  apply_terms(m.terms, T(1), true);  return *this;
        }
        template <class E> const vector& operator+=(const mixed_expression<E, T> &m) {
            if (inlinable(m.terms)) { detail::assign_expression<assign::ADD>(*this, detail::fused_mixed<E, T>(m.expr, m.terms, T(1))); return *this; }
            *this += m.expr; apply_terms(m.terms, T(1), true);  return *this;
        }
        template <class E> const vector& operator-=(const mixed_expression<E, T> &m) {
            if (inlinable(m.terms)) { detail::assign_expression<assign::SUB>(*this, detail::fused_mixed<E, T>(m.expr, m.terms, T(1))); return *this; }
            *this -= m.expr; apply_terms(m.terms, T(-1), true); return *this;
        }

        // ---- expression terminal protocol -------------------------------------------------
        int lower(detail::ir_builder &b) const { b.push_vec(buf[b.part].raw(), dtype_of<T>::value); return dtype_of<T>::value; }
        void props(detail::expr_props &p) const { p.see(queue, part, size()); }

        // ---- host <-> device (vector.hpp:805-911) -----------------------------------------
        void write_data(size_t offset, size_t size, const T *hostptr, bool blocking) {
            if (!size) return;
            for (unsigned d = 0; d < queue.size(); ++d) {
                size_t start = std::max(offset, part[d]), stop = std::min(offset + size, part[d + 1]);
                if (stop <= start) continue;
                buf[d].write(queue[d], start - part[d], stop - start, hostptr + start - offset, false);
            }
            if (blocking) for (unsigned d = 0; d < queue.size(); ++d) queue[d].finish();
        }
        void read_data(size_t offset, size_t size, T *hostptr, bool blocking) const {
            if (!size) return;
            for (unsigned d = 0; d < queue.size(); ++d) {
                size_t start = std::max(offset, part[d]), stop = std::min(offset + size, part[d + 1]);
                if (stop <= start) continue;
                buf[d].read(queue[d], start - part[d], stop - start, hostptr + start - offset, false);
            }
            if (blocking) for (unsigned d = 0; d < queue.size(); ++d) queue[d].finish();
        }
    private:
        std::vector<backend::command_queue> queue;
        std::vector<size_t> part;
        std::vector<backend::device_vector<T>> buf;

        void allocate_buffers(backend::mem_flags flags, const T *host) {                 // vector.hpp:918-928
            for (unsigned d = 0; d < queue.size(); ++d)
                buf[d] = backend::device_vector<T>(queue[d], part[d + 1] - part[d], host ? host + part[d] : static_cast<const T*>(0), flags);
        }
        void apply_terms(const detail::additive_terms<T> &a, T sign, bool append) {
            for (auto &t : a.terms) { t(*this, sign, append); append = true; }
        }
        bool inlinable(const detail::additive_terms<T> &a) const {
            if (a.terms.empty() || a.terms.size() > 6 || !std::is_floating_point<T>::value) return false;
            // a term is inlined thread per row, or -- one distinct sliced-ELL matrix per assignment -- by a storage-order sweep
            const vexb_spmat *swept = nullptr;
            for (auto &t : a.terms) for (unsigned d = 0; d < queue.size(); ++d) {
                if (t.can_inline(d)) continue;
                if (!t.sweep_strip(d) || (swept && swept != t.sweep_strip(0))) return false;
                swept = t.sweep_strip(0);
            }
            return true;
        }
};

template <typename T> void swap(vector<T> &x, vector<T> &y) { x.swap(y); }

// ---- copy() family (vector.hpp:998-1228) ---------------------------------------------------
template <class T> void copy(const vector<T> &dv, T *hv, bool blocking = true) { dv.read_data(0, dv.size(), hv, blocking); }
template <class T> void copy(const T *hv, vector<T> &dv, bool blocking = true) { dv.write_data(0, dv.size(), hv, blocking); }
template <class T> void copy(const vector<T> &dv, std::vector<T> &hv, bool blocking = true) {
    precondition(dv.size() == hv.size(), "vex::copy: sizes differ"); dv.read_data(0, dv.size(), hv.data(), blocking);
}
template <class T> void copy(const std::vector<T> &hv, vector<T> &dv, bool blocking = true) {
    precondition(dv.size() == hv.size(), "vex::copy: sizes differ"); dv.write_data(0, dv.size(), hv.data(), blocking);
}
template <class T> void copy(const vector<T> &src, vector<T> &dst) { dst = src; }
// explicit-queue forms (the queue list is that of the device vector)
template <class T> void copy(const std::vector<backend::command_queue>&, const vector<T> &dv, T *hv, bool blocking = true) { copy(dv, hv, blocking); }
template <class T> void copy(const std::vector<backend::command_queue>&, const T *hv, vector<T> &dv, bool blocking = true) { copy(hv, dv, blocking); }
// type-converting forms go through a temporary
template <class T, class H> typename std::enable_if<!std::is_same<T, H>::value>::type
copy(const vector<T> &dv, std::vector<H> &hv, bool blocking = true) { std::vector<T> t(dv.size()); copy(dv, t, true); (void)blocking; hv.assign(t.begin(), t.end()); }
template <class T, class H> typename std::enable_if<!std::is_same<T, H>::value>::type
copy(const std::vector<H> &hv, vector<T> &dv, bool blocking = true) { std::vector<T> t(hv.begin(), hv.end()); copy(t, dv, blocking); }
// iterator-range forms
template <class V, class OutputIterator>
typename std::enable_if<std::is_pointer<OutputIterator>::value || std::is_class<OutputIterator>::value, OutputIterator>::type
copy(const typename vector<V>::const_iterator &first, const typename vector<V>::const_iterator &last, OutputIterator result, bool blocking = true) {
    std::vector<V> t(last - first);
    first.vec->read_data(first.pos, t.size(), t.data(), true); (void)blocking;
    return std::copy(t.begin(), t.end(), result);
}
template <class T> T* copy(typename vector<T>::const_iterator first, typename vector<T>::const_iterator last, T *result, bool blocking = true) {
    first.vec->read_data(first.pos, last - first, result, blocking); return result + (last - first);
}
template <class T> T* copy(typename vector<T>::iterator first, typename vector<T>::iterator last, T *result, bool blocking = true) {
    first.vec->read_data(first.pos, last - first, result, blocking); return result + (last - first);
}
template <class T> typename vector<T>::iterator copy(const T *first, const T *last, typename vector<T>::iterator result, bool blocking = true) {
    result.vec->write_data(result.pos, last - first, first, blocking); return result + (last - first);
}
template <class T> typename vector<T>::iterator
copy(typename std::vector<T>::const_iterator first, typename std::vector<T>::const_iterator last, typename vector<T>::iterator result, bool blocking = true) {
    result.vec->write_data(result.pos, last - first, &*first, blocking); return result + (last - first);
}

/// 1 / time of `a = b + c` on 1M floats, second run (vector.hpp:1237-1255).
inline double device_vector_perf(const backend::command_queue &q) {
    static const size_t test_size = 1024U * 1024U;
    std::vector<backend::command_queue> queue(1, q);
    vex::vector<float> a(queue, test_size), b(queue, test_size), c(queue, test_size);
    b = 1.0f; c = 2.0f;
    a = b + c;
    profiler<> prof(queue);
    prof.tic_cl("");
    a = b + c;
    return 1.0 / prof.toc("");
}

template <class T>
std::ostream& operator<<(std::ostream &o, const vex::vector<T> &t) {
    std::vector<T> h(t.size());
    copy(t, h);
    o << "{";
    for (size_t i = 0; i < h.size(); ++i) { if (i % 10 == 0) o << "\n" << std::setw(6) << i << ":"; o << " " << h[i]; }
    return o << "\n}\n";
}

} // namespace vex
#endif
