#ifndef VEXCL_REDUCE_BY_KEY_HPP
#define VEXCL_REDUCE_BY_KEY_HPP
// vex::reduce_by_key with the reference's spelling (vexcl/reduce_by_key.hpp:569-581) and its default operators: keys
// compare with ==, values add.  It resizes okeys and ovals to the number of runs of equal keys and returns that number;
// okeys[j] holds the bits of the last key of run j (the reference's key_value_mapping), ovals[j] the sum of its values
// in an order that depends on n only.  -0.0 and +0.0 share a run; every NaN key is a run of its own.  After
// vex::sort_by_key it is a group-by.  One part only, as in the reference; two calls to the library (vexb_reduce_by_key_count
// returns the count after two launches and one read, vexb_reduce_by_key_write writes the runs in a third).  Other
// comparators or operators and tuples of keys stop at a static_assert.
#include <type_traits>
#include "scan_by_key.hpp"

namespace vex {

/// Reduce by key: one (last key, sum of values) per run of equal keys; returns the number of runs.
template <typename K, typename V>
int reduce_by_key(const vector<K> &ikeys, const vector<V> &ivals, vector<K> &okeys, vector<V> &ovals) {
    static_assert(detail::sortable<K>::value && detail::sortable<V>::value,
                  "vex::reduce_by_key takes keys and values of double, float, int, unsigned and 64-bit integers");
    precondition(ikeys.nparts() == 1 && ivals.nparts() == 1, "reduce_by_key is only supported for single device contexts");
    precondition(ikeys.size() == ivals.size(), "keys and values should have same size");
    precondition(static_cast<const void *>(&okeys) != static_cast<const void *>(&ikeys) &&
                 static_cast<const void *>(&ovals) != static_cast<const void *>(&ivals),
                 "reduce_by_key writes okeys and ovals apart from its inputs");
    const auto &queue = ikeys.queue_list();
    const size_t n = ikeys.size();
    size_t bytes = 0, runs = 0;
    backend::device_vector<char> ws = detail::scan_workspace<V>(queue[0], n, &bytes);
    const int kdt = dtype_of<K>::value, vdt = dtype_of<V>::value;
    if (n)
        VEXB_CHECKED(vexb_reduce_by_key_count(queue[0].ordinal(), queue[0].raw(), ikeys(0).raw(), kdt, ivals(0).raw(), vdt,
                                              n, ws.raw(), bytes, &runs));
    okeys.resize(queue, runs);
    ovals.resize(queue, runs);
    if (n)
        VEXB_CHECKED(vexb_reduce_by_key_write(queue[0].ordinal(), queue[0].raw(), ikeys(0).raw(), kdt, ivals(0).raw(), vdt,
                                              n, okeys(0).raw(), ovals(0).raw(), ws.raw(), bytes));
    return static_cast<int>(runs);
}

/// Reduce by key with another comparator or operator (VEX_FUNCTION, VEX_DUAL_FUNCTOR), or of tuples of keys.
template <class IKeys, class OKeys, typename V, class Comp, class Oper>
int reduce_by_key(IKeys &&, const vector<V> &, OKeys &&, vector<V> &, Comp, Oper) {
    static_assert(detail::scan_unsupported<Comp>::value, VEXCL_SCAN_OPERATOR_MESSAGE);
    return 0;
}
template <class IKeys, class OKeys, typename V,
          class = typename std::enable_if<!detail::is_vex_vector<typename std::decay<IKeys>::type>::value>::type>
int reduce_by_key(IKeys &&, const vector<V> &, OKeys &&, vector<V> &) {
    static_assert(detail::scan_unsupported<IKeys>::value, VEXCL_SCAN_OPERATOR_MESSAGE);
    return 0;
}

} // namespace vex
#endif
