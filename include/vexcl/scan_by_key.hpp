#ifndef VEXCL_SCAN_BY_KEY_HPP
#define VEXCL_SCAN_BY_KEY_HPP
// vex::inclusive_scan_by_key and vex::exclusive_scan_by_key with the reference's spellings
// (vexcl/scan_by_key.hpp:736-758) and its default operators: keys compare with ==, values add.  A run is a maximal
// range of equal keys: -0.0 and +0.0 share one, and every NaN key is a run of its own.  Keys and values are vectors of
// double, float, int, unsigned, 64-bit signed or unsigned integers in any combination, on one part, scanned by the
// library's reduce-then-scan kernels (vexb_scan_by_key, three launches).
//
// inclusive_scan_by_key ignores init, as the reference's kernel does; exclusive_scan_by_key starts every run at init.
// ovals may be ivals (in place); keys must not be ovals.  Vectors of several parts throw, as in the reference.  Other
// comparators or operators and tuples of keys need a generated kernel; they stop at a static_assert.
#include <type_traits>
#include "scan.hpp"

namespace vex {

namespace detail {

template <class K, class V>
void scan_by_key_part(const vector<K> &keys, const vector<V> &ivals, vector<V> &ovals, V init, bool exclusive) {
    static_assert(sortable<K>::value && sortable<V>::value,
                  "vex scans by key take keys and values of double, float, int, unsigned and 64-bit integers");
    precondition(keys.nparts() == 1 && ivals.nparts() == 1, "scan_by_key is only supported for single device contexts");
    precondition(ivals.size() == ovals.size() && ivals.nparts() == ovals.nparts(), "input and output should have same size");
    precondition(keys.size() == ivals.size(), "keys and values should have same size");
    const size_t n = keys.size();
    if (!n) return;
    const auto &q = keys.queue_list()[0];
    size_t bytes = 0;
    backend::device_vector<char> ws = scan_workspace<V>(q, n, &bytes);
    VEXB_CHECKED(vexb_scan_by_key(q.ordinal(), q.raw(), keys(0).raw(), dtype_of<K>::value, ivals(0).raw(), ovals(0).raw(),
                                  dtype_of<V>::value, n, exclusive, &init, ws.raw(), bytes));
}

template <class K> struct is_vex_vector : std::false_type {};
template <class T> struct is_vex_vector<vector<T>> : std::true_type {};

} // namespace detail

/// Inclusive scan by key: the sum of the values from the head of each run of equal keys.  init is not read.
template <typename K, typename V>
void inclusive_scan_by_key(const vector<K> &keys, const vector<V> &ivals, vector<V> &ovals, V init = V()) {
    detail::scan_by_key_part(keys, ivals, ovals, init, false);
}

/// Exclusive scan by key: every run of equal keys starts at init.
template <typename K, typename V>
void exclusive_scan_by_key(const vector<K> &keys, const vector<V> &ivals, vector<V> &ovals, V init = V()) {
    detail::scan_by_key_part(keys, ivals, ovals, init, true);
}

/// Scans with another comparator or operator (VEX_FUNCTION, VEX_DUAL_FUNCTOR), or of tuples of keys.
template <class K, typename V, class Comp, class Oper>
void inclusive_scan_by_key(K &&, const vector<V> &, vector<V> &, Comp, Oper, V = V()) {
    static_assert(detail::scan_unsupported<Comp>::value, VEXCL_SCAN_OPERATOR_MESSAGE);
}
template <class K, typename V, class Comp, class Oper>
void exclusive_scan_by_key(K &&, const vector<V> &, vector<V> &, Comp, Oper, V = V()) {
    static_assert(detail::scan_unsupported<Comp>::value, VEXCL_SCAN_OPERATOR_MESSAGE);
}
template <class K, typename V, class = typename std::enable_if<!detail::is_vex_vector<typename std::decay<K>::type>::value>::type>
void inclusive_scan_by_key(K &&, const vector<V> &, vector<V> &, V = V()) {
    static_assert(detail::scan_unsupported<K>::value, VEXCL_SCAN_OPERATOR_MESSAGE);
}
template <class K, typename V, class = typename std::enable_if<!detail::is_vex_vector<typename std::decay<K>::type>::value>::type>
void exclusive_scan_by_key(K &&, const vector<V> &, vector<V> &, V = V()) {
    static_assert(detail::scan_unsupported<K>::value, VEXCL_SCAN_OPERATOR_MESSAGE);
}

} // namespace vex
#endif
