// vex::sort and vex::sort_by_key: the reference's tests/sort.cpp cases sort_keys and sort_keys_vals_default (only the
// Boost.Test harness replaced), then greater, less_equal and greater_equal checked in full against std::stable_sort,
// and keys and values partitioned differently, which throws.
#include "testing.hpp"
#include <algorithm>
#include <vexcl/vector.hpp>
#include <vexcl/sort.hpp>

BOOST_AUTO_TEST_CASE(sort_keys)
{
    const size_t n = 1000 * 1000;

    std::vector<float> k = random_vector<float>(n);
    vex::vector<float> keys(ctx, k);

    vex::sort(keys);
    vex::copy(keys, k);

    BOOST_CHECK( std::is_sorted(k.begin(), k.end()) );
}

BOOST_AUTO_TEST_CASE(sort_keys_vals_default)
{
    const size_t n = 1000 * 1000;

    std::vector<int  > k = random_vector<int  >(n);
    std::vector<float> v = random_vector<float>(n);
    std::vector<int>   p(n);

    vex::vector<int  > keys(ctx, k);
    vex::vector<float> vals(ctx, v);

    for(size_t i = 0; i < p.size(); ++i) p[i] = static_cast<int>(i);
    std::stable_sort(p.begin(), p.end(), [&](int i, int j) { return k[i] < k[j]; });

    vex::sort_by_key(keys, vals);

    check_sample(keys, [&](size_t pos, int val) {
            BOOST_CHECK_EQUAL(val, k[p[pos]]);
            });

    check_sample(vals, [&](size_t pos, float val) {
            BOOST_CHECK_EQUAL(val, v[p[pos]]);
            });
}

// Every element: keys and values after sort_by_key(keys, vals, comp) equal std::stable_sort's with the host comparator.
template <class K, class Comp>
void check_full(Comp comp, size_t n) {
    std::vector<K> k = random_vector<K>(n);
    std::vector<long long> v(n);
    for (size_t i = 0; i < n; ++i) v[i] = static_cast<long long>(i);
    std::vector<size_t> p(n);
    for (size_t i = 0; i < n; ++i) p[i] = i;
    // the stable order of a non-strict comparator is taken to be that of its strict counterpart
    std::stable_sort(p.begin(), p.end(), [&](size_t i, size_t j) { return comp(k[i], k[j]) && !comp(k[j], k[i]); });

    vex::vector<K> keys(ctx, k);
    vex::vector<long long> vals(ctx, v);
    vex::sort_by_key(keys, vals, comp);
    std::vector<K> gk(n);
    std::vector<long long> gv(n);
    vex::copy(keys, gk);
    vex::copy(vals, gv);
    bool same = true;
    for (size_t i = 0; i < n; ++i) same = same && gk[i] == k[p[i]] && gv[i] == static_cast<long long>(p[i]);
    BOOST_CHECK(same);

    vex::vector<K> alone(ctx, k);
    vex::sort(alone, comp);
    vex::copy(alone, gk);
    same = true;
    for (size_t i = 0; i < n; ++i) same = same && gk[i] == k[p[i]];
    BOOST_CHECK(same);
}

BOOST_AUTO_TEST_CASE(sort_greater)
{
    check_full<int>(vex::greater<int>(), 1000 * 1000);
    check_full<double>(vex::greater<double>(), 300 * 1000);
}

BOOST_AUTO_TEST_CASE(sort_less_equal)
{
    check_full<unsigned>(vex::less_equal<unsigned>(), 1000 * 1000);
    check_full<float>(vex::less_equal<float>(), 300 * 1000);
}

BOOST_AUTO_TEST_CASE(sort_greater_equal)
{
    check_full<long long>(vex::greater_equal<long long>(), 1000 * 1000);
    check_full<unsigned long long>(vex::greater_equal<unsigned long long>(), 5);
}

BOOST_AUTO_TEST_CASE(sort_keys_vals_partitioned_differently)
{
    std::vector<vex::command_queue> one(1, ctx.queue(0));
    vex::vector<int> keys(ctx, 1000);
    vex::vector<int> vals(one, 1000);
    if (ctx.size() > 1)
        BOOST_CHECK_THROW(vex::sort_by_key(keys, vals), std::runtime_error);
    vex::vector<int> fewer(ctx, 999);
    BOOST_CHECK_THROW(vex::sort_by_key(keys, fewer), std::runtime_error);
}
