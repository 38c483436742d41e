#ifndef VEXCL_SCAN_HPP
#define VEXCL_SCAN_HPP
// vex::inclusive_scan and vex::exclusive_scan with the reference's spellings (vexcl/scan.hpp:426-518) and its one
// operator, vex::plus<T>.  Elements are double, float, int, unsigned, 64-bit signed or unsigned integers.  Each part is
// scanned on its own queue by the library's reduce-then-scan kernels (vexb_scan, three launches); integer sums wrap and
// every float add is rounded on its own, in an order that depends on the part's size only.
//
// inclusive_scan ignores init, as the reference's kernels do.  exclusive_scan writes init, with its own bits, to out[0].
// With several parts, one boundary value per part is read, the carries are folded on the host in T, and each carry is
// added to its part with one launch of the expression path.  init is counted once; the reference counts it once for
// every part up to the current one.
//
// Other operators (VEX_FUNCTION, VEX_DUAL_FUNCTOR or any functor but vex::plus<T>) need a generated kernel this back
// end does not have; they stop at a static_assert.
#include <cstring>
#include <functional>
#include <type_traits>
#include <vector>
#include "backend.hpp"
#include "util.hpp"
#include "types.hpp"
#include "vector.hpp"
#include "sort.hpp"

namespace vex {

/// Function object class for addition: the scans' only operator.
template <typename T> struct plus : std::plus<T> { plus() {} };

namespace detail {

template <class T> struct scan_unsupported : std::false_type {};

#define VEXCL_SCAN_OPERATOR_MESSAGE \
    "vex scans and reduce_by_key support only vex::plus<T> on the values and == on the keys of a vex::vector<K>"

/// The exact identity of T's add: -0.0 for floats (-0.0 + x == x, also for x = +0.0), 0 for integers.
template <class T> T scan_identity() { return std::is_floating_point<T>::value ? -T(0) : T(0); }

/// a + b in T; integers wrap.
template <class T> T scan_add(T a, T b) {
    if constexpr (std::is_integral<T>::value) {
        typedef typename std::make_unsigned<T>::type U;
        const U s = static_cast<U>(static_cast<U>(a) + static_cast<U>(b));
        T r;
        std::memcpy(&r, &s, sizeof(T));
        return r;
    } else {
        return a + b;
    }
}

/// Workspace of vexb_scan / vexb_scan_by_key / vexb_reduce_by_key_* for n elements of V on queue q.
template <class V>
backend::device_vector<char> scan_workspace(const backend::command_queue &q, size_t n, size_t *bytes) {
    VEXB_CHECKED(vexb_scan_workspace_bytes(n, dtype_of<V>::value, bytes));
    return backend::device_vector<char>(q, *bytes);
}

template <class T>
void scan_parts(const vector<T> &input, vector<T> &output, T init, bool exclusive) {
    static_assert(sortable<T>::value, "vex scans take vectors of double, float, int, unsigned and 64-bit integers");
    precondition(input.nparts() == output.nparts() && input.partition() == output.partition(), "Incompatible partitioning");
    const auto &queue = input.queue_list();
    const int dt = dtype_of<T>::value;
    const T ident = scan_identity<T>();
    // an exclusive scan in place overwrites each part's last input, which its carry needs: read those first
    std::vector<T> last_in(queue.size());
    if (exclusive && queue.size() > 1)
        for (unsigned d = 0; d < queue.size(); ++d)
            if (size_t n = input.part_size(d)) input(d).read(queue[d], n - 1, 1, &last_in[d], true);
    bool started = false;
    for (unsigned d = 0; d < queue.size(); ++d) {
        const size_t n = input.part_size(d);
        if (!n) continue;
        size_t bytes = 0;
        backend::device_vector<char> ws = scan_workspace<T>(queue[d], n, &bytes);
        VEXB_CHECKED(vexb_scan(queue[d].ordinal(), queue[d].raw(), input(d).raw(), output(d).raw(), dt, n, exclusive,
                               started ? &ident : &init, ws.raw(), bytes));
        started = true;
    }
    if (queue.size() <= 1) return;
    // the parts' local totals, folded on the host in T; each carry is added to its part (scan.hpp:444-458)
    T carry = ident;
    bool have = false;
    for (unsigned d = 0; d < queue.size(); ++d) {
        const size_t n = output.part_size(d);
        if (!n) continue;
        T total;
        output(d).read(queue[d], n - 1, 1, &total, true);
        if (exclusive) total = scan_add(total, last_in[d]);
        if (have) {
            vector<T> part(queue[d], output(d), n);
            part += carry;
            carry = scan_add(carry, total);
        } else {
            carry = total;
            have = true;
        }
    }
}

} // namespace detail

/// Inclusive scan: output[i] = input[0] + ... + input[i].  init is not read, as in the reference.
template <typename T, class Oper>
void inclusive_scan(const vector<T> &input, vector<T> &output, T init, Oper) {
    static_assert(std::is_same<Oper, plus<T>>::value, VEXCL_SCAN_OPERATOR_MESSAGE);
    detail::scan_parts(input, output, init, false);
}

/// Inclusive scan: output[i] = input[0] + ... + input[i].  init is not read, as in the reference.
template <typename T>
void inclusive_scan(const vector<T> &input, vector<T> &output, T init = T()) {
    inclusive_scan(input, output, init, plus<T>());
}

/// Exclusive scan: output[0] = init, output[i] = init + input[0] + ... + input[i - 1].
template <typename T, class Oper>
void exclusive_scan(const vector<T> &input, vector<T> &output, T init, Oper) {
    static_assert(std::is_same<Oper, plus<T>>::value, VEXCL_SCAN_OPERATOR_MESSAGE);
    detail::scan_parts(input, output, init, true);
}

/// Exclusive scan: output[0] = init, output[i] = init + input[0] + ... + input[i - 1].
template <typename T>
void exclusive_scan(const vector<T> &input, vector<T> &output, T init = T()) {
    exclusive_scan(input, output, init, plus<T>());
}

} // namespace vex
#endif
