#ifndef VEXCL_SORT_HPP
#define VEXCL_SORT_HPP
// vex::sort and vex::sort_by_key with the reference's spellings (vexcl/sort.hpp:2120-2182), for the built-in
// comparators over the key type: vex::less and vex::less_equal sort ascending, vex::greater and vex::greater_equal
// descending.  Keys are vector<T> of double, float, int, unsigned, 64-bit signed or unsigned integers; values one vector
// of any of those types.  Each part is sorted on its own queue by the library's radix sort (vexb_sort); a vector of
// several parts is then read back, merged on the host (vexb_sort_merge) and written back, as the reference does.
//
// The sort is stable in both directions.  less_equal and greater_equal are not strict orders and the reference leaves
// their order of equal keys open; here they give exactly the output of less and greater.  Floating keys: -0.0 equals
// +0.0, NaNs equal each other and are greater than +inf, so ascending puts them last and descending first.
//
// Comparators written with VEX_FUNCTION or VEX_DUAL_FUNCTOR, and tuples of keys or values, need a comparison sort this
// back end does not generate; they stop at a static_assert.
#include <functional>
#include <type_traits>
#include <vector>
#include "backend.hpp"
#include "util.hpp"
#include "types.hpp"
#include "vector.hpp"

namespace vex {

/// Function object class for less-than inequality comparison.
template <typename T> struct less : std::less<T> { less() {} };
/// Function object class for less-than-or-equal inequality comparison.
template <typename T> struct less_equal : std::less_equal<T> { less_equal() {} };
/// Function object class for greater-than inequality comparison.
template <typename T> struct greater : std::greater<T> { greater() {} };
/// Function object class for greater-than-or-equal inequality comparison.
template <typename T> struct greater_equal : std::greater_equal<T> { greater_equal() {} };

namespace detail {

template <class T> struct sortable : std::integral_constant<bool,
    std::is_same<T, double>::value || std::is_same<T, float>::value || std::is_same<T, int>::value ||
    std::is_same<T, unsigned>::value || std::is_same<T, long>::value || std::is_same<T, unsigned long>::value ||
    std::is_same<T, long long>::value || std::is_same<T, unsigned long long>::value> {};

template <class Comp, class K> struct sort_direction { static const bool supported = false, descending = false; };
template <class K> struct sort_direction<less<K>, K>          { static const bool supported = true, descending = false; };
template <class K> struct sort_direction<less_equal<K>, K>    { static const bool supported = true, descending = false; };
template <class K> struct sort_direction<greater<K>, K>       { static const bool supported = true, descending = true; };
template <class K> struct sort_direction<greater_equal<K>, K> { static const bool supported = true, descending = true; };

template <class K, class V, class Comp>
void sort_parts(vector<K> &keys, vector<V> *vals, Comp) {
    static_assert(sort_direction<Comp, K>::supported,
                  "vex::sort / vex::sort_by_key support only vex::less<K>, vex::less_equal<K>, vex::greater<K> and "
                  "vex::greater_equal<K> over the key type K of a vex::vector<K>");
    static_assert(sortable<K>::value && sortable<V>::value,
                  "vex::sort / vex::sort_by_key take keys and values of double, float, int, unsigned and 64-bit integers");
    const int desc = sort_direction<Comp, K>::descending;
    const int kdt = dtype_of<K>::value, vdt = vals ? dtype_of<V>::value : -1;
    const auto &queue = keys.queue_list();
    precondition(!vals || (vals->nparts() == keys.nparts() && vals->partition() == keys.partition()),
                 "Keys and values span different devices");
    for (unsigned d = 0; d < queue.size(); ++d) {
        const size_t n = keys.part_size(d);
        if (!n) continue;
        size_t bytes = 0;
        VEXB_CHECKED(vexb_sort_workspace_bytes(n, kdt, vdt, &bytes));
        backend::device_vector<char> ws(queue[d], bytes);
        VEXB_CHECKED(vexb_sort(queue[d].ordinal(), queue[d].raw(), keys(d).raw(), kdt, vals ? (*vals)(d).raw() : nullptr,
                               vdt, n, desc, ws.raw(), bytes));
    }
    if (queue.size() <= 1) return;
    // the parts are sorted on their devices; merge them on the host (sort.hpp:2081-2087)
    std::vector<K> hk(keys.size()), ok(keys.size());
    std::vector<V> hv(vals ? keys.size() : 0), ov(hv.size());
    copy(keys, hk);
    if (vals) copy(*vals, hv);
    VEXB_CHECKED(vexb_sort_merge(static_cast<int>(queue.size()), keys.partition().data(), hk.data(), kdt,
                                 vals ? hv.data() : nullptr, vdt, desc, ok.data(), vals ? ov.data() : nullptr));
    copy(ok, keys);
    if (vals) copy(ov, *vals);
}

} // namespace detail

/// Sorts the vector in the order of comp (vex::less, vex::less_equal, vex::greater or vex::greater_equal over K).
template <class K, class Comp>
void sort(vector<K> &keys, Comp comp) {
    detail::sort_parts<K, K>(keys, nullptr, comp);
}

/// Sorts the vector into ascending order.
template <class K>
void sort(vector<K> &keys) {
    sort(keys, less<K>());
}

/// Sorts keys in the order of comp and moves the values with them; equal keys keep their order.
template <class K, class V, class Comp>
void sort_by_key(vector<K> &keys, vector<V> &vals, Comp comp) {
    detail::sort_parts(keys, &vals, comp);
}

/// Sorts the elements in keys and values into ascending key order.
template <class K, class V>
void sort_by_key(vector<K> &keys, vector<V> &vals) {
    sort_by_key(keys, vals, less<K>());
}

/// Tuples of keys or values (boost::fusion sequences in the reference) need a comparison sort this back end lacks.
template <class K, class Comp>
void sort(K &&, Comp) {
    static_assert(sizeof(K) == 0, "vex::sort / vex::sort_by_key support only vex::less<K>, vex::less_equal<K>, "
                  "vex::greater<K> and vex::greater_equal<K> over the key type K of a vex::vector<K>");
}
template <class K, class V, class Comp>
void sort_by_key(K &&, V &&, Comp) {
    static_assert(sizeof(K) == 0, "vex::sort / vex::sort_by_key support only vex::less<K>, vex::less_equal<K>, "
                  "vex::greater<K> and vex::greater_equal<K> over the key type K of a vex::vector<K>");
}

} // namespace vex
#endif
