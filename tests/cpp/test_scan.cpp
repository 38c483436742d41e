// vex::inclusive_scan, vex::exclusive_scan, vex::inclusive_scan_by_key, vex::exclusive_scan_by_key and
// vex::reduce_by_key: the reference's tests/scan.cpp cases inclusive and exclusive, tests/scan_by_key.cpp's sbk and
// tests/reduce_by_key.cpp's rbk (only the Boost.Test harness replaced), then vex::sort_by_key followed by
// vex::reduce_by_key against a host group-by, exclusive_scan counting init once across parts, and the refusals.
#include "testing.hpp"
#include <algorithm>
#include <map>
#include <numeric>
#include <vexcl/vector.hpp>
#include <vexcl/scan.hpp>
#include <vexcl/scan_by_key.hpp>
#include <vexcl/reduce_by_key.hpp>
#include <vexcl/sort.hpp>

BOOST_AUTO_TEST_CASE(inclusive)
{
    const size_t n = 1000 * 1000;

    std::vector<int> x = random_vector<int>(n);
    vex::vector<int> X(ctx, x);

    vex::inclusive_scan(X, X);

    std::partial_sum(x.begin(), x.end(), x.begin());

    check_sample(X, [&](size_t idx, int v) {
            BOOST_CHECK_EQUAL(v, x[idx]);
            });
}

BOOST_AUTO_TEST_CASE(exclusive)
{
    const size_t n = 1000 * 1000;

    std::vector<double> x = random_vector<double>(n);
    vex::vector<double> X(ctx, x);

    vex::exclusive_scan(X, X);

    std::partial_sum(x.begin(), x.end(), x.begin());
    std::rotate(x.rbegin(), x.rbegin() + 1, x.rend());
    x[0] = 0;

    check_sample(X, [&](size_t idx, double v) {
            BOOST_CHECK_CLOSE(v, x[idx], 1e-8f);
            });
}

BOOST_AUTO_TEST_CASE(sbk)
{
    const int n = 1000;

    std::vector<int> x = random_vector<int>(n);
    std::vector<int> y = random_vector<int>(n);

    std::sort(x.begin(), x.end());

    std::vector<vex::backend::command_queue> queue(1, ctx.queue(0));

    vex::vector<int> ikeys(queue, x);
    vex::vector<int> ivals(queue, y);
    vex::vector<int> ovals(queue, n);

    vex::inclusive_scan_by_key(ikeys, ivals, ovals);

    check_sample(ovals, [&](size_t i, int v) {
            if (i == 0)
                BOOST_CHECK_EQUAL(v, y[i]);
            else if (x[i-1] == x[i])
                BOOST_CHECK_EQUAL(
                    y[i],
                    static_cast<int>(ovals[i]) - static_cast<int>(ovals[i-1])
                    );
            else
                BOOST_CHECK_EQUAL(v, y[i]);
            });

    vex::exclusive_scan_by_key(ikeys, ivals, ovals);

    check_sample(ovals, [&](size_t i, int v) {
            if (i == 0)
                BOOST_CHECK_EQUAL(v, 0);
            else if (x[i-1] == x[i])
                BOOST_CHECK_EQUAL(
                    y[i-1],
                    static_cast<int>(ovals[i]) - static_cast<int>(ovals[i-1])
                    );
            else
                BOOST_CHECK_EQUAL(v, 0);
            });
}

BOOST_AUTO_TEST_CASE(rbk)
{
    const int n = 1024 * 1024;

    std::vector<int>    x = random_vector<int>   (n);
    std::vector<double> y = random_vector<double>(n);

    std::sort(x.begin(), x.end());

    std::vector<vex::backend::command_queue> queue(1, ctx.queue(0));

    vex::vector<int>    ikeys(queue, x);
    vex::vector<double> ivals(queue, y);

    vex::vector<int>    okeys;
    vex::vector<double> ovals;

    int num_keys = vex::reduce_by_key(ikeys, ivals, okeys, ovals);

    std::vector<int> ux = x;
    ux.erase( std::unique(ux.begin(), ux.end()), ux.end() );

    BOOST_CHECK_EQUAL(ux.size(),    num_keys);
    BOOST_CHECK_EQUAL(okeys.size(), num_keys);
    BOOST_CHECK_EQUAL(ovals.size(), num_keys);

    check_sample(okeys, ovals, [&](size_t, int key, double dev_sum) {
        double host_sum = std::accumulate(
                y.begin() + (std::lower_bound(x.begin(), x.end(), key) - x.begin()),
                y.begin() + (std::upper_bound(x.begin(), x.end(), key) - x.begin()),
                0.0);
        BOOST_CHECK_CLOSE(dev_sum, host_sum, 1e-8);
        });
}

// Every element: sort_by_key then reduce_by_key is a group-by, checked against std::map sums (exact for integers).
BOOST_AUTO_TEST_CASE(sort_then_reduce_by_key)
{
    const size_t n = 2 * 1000 * 1000 + 5;
    std::vector<vex::backend::command_queue> queue(1, ctx.queue(0));
    std::vector<unsigned> k(n);
    std::vector<long long> v(n);
    std::default_random_engine rng(42);
    std::uniform_int_distribution<unsigned> key(0, 50000);
    std::uniform_int_distribution<long long> val(-1000000, 1000000);
    std::map<unsigned, long long> sums;
    for (size_t i = 0; i < n; ++i) { k[i] = key(rng); v[i] = val(rng); sums[k[i]] += v[i]; }

    vex::vector<unsigned> keys(queue, k);
    vex::vector<long long> vals(queue, v);
    vex::sort_by_key(keys, vals);
    vex::vector<unsigned> okeys;
    vex::vector<long long> ovals;
    int m = vex::reduce_by_key(keys, vals, okeys, ovals);
    BOOST_REQUIRE(static_cast<size_t>(m) == sums.size());
    std::vector<unsigned> gk(m);
    std::vector<long long> gv(m);
    vex::copy(okeys, gk);
    vex::copy(ovals, gv);
    bool same = true;
    size_t j = 0;
    for (const auto &kv : sums) { same = same && gk[j] == kv.first && gv[j] == kv.second; ++j; }
    BOOST_CHECK(same);
}

// exclusive_scan with init on every context (two parts unless VEXCL_TEST_PARTS=1): init is counted once.
BOOST_AUTO_TEST_CASE(exclusive_init_once)
{
    const size_t n = 100 * 1000 + 3;
    std::vector<long long> x(n);
    for (size_t i = 0; i < n; ++i) x[i] = static_cast<long long>(i % 1000) - 500;
    vex::vector<long long> X(ctx, x), Y(ctx, n);
    vex::exclusive_scan(X, Y, 1000000LL);
    vex::inclusive_scan(X, X, 5LL);
    std::vector<long long> gy(n), gx(n);
    vex::copy(Y, gy);
    vex::copy(X, gx);
    long long s = 0;
    bool same = true;
    for (size_t i = 0; i < n; ++i) {
        same = same && gy[i] == 1000000LL + s;
        s += x[i];
        same = same && gx[i] == s;
    }
    BOOST_CHECK(same);
}

BOOST_AUTO_TEST_CASE(refusals)
{
    vex::vector<int> keys(ctx, 1000), okeys;
    vex::vector<double> vals(ctx, 1000), ovals;
    if (ctx.size() > 1) {
        BOOST_CHECK_THROW(vex::inclusive_scan_by_key(keys, vals, vals), std::runtime_error);
        BOOST_CHECK_THROW(vex::exclusive_scan_by_key(keys, vals, vals), std::runtime_error);
        BOOST_CHECK_THROW(vex::reduce_by_key(keys, vals, okeys, ovals), std::runtime_error);
    }
    std::vector<vex::backend::command_queue> queue(1, ctx.queue(0));
    vex::vector<int> k1(queue, 1000);
    vex::vector<double> v1(queue, 1000), fewer(queue, 999);
    BOOST_CHECK_THROW(vex::inclusive_scan_by_key(k1, v1, fewer), std::runtime_error);
    BOOST_CHECK_THROW(vex::reduce_by_key(k1, fewer, okeys, ovals), std::runtime_error);
    vex::vector<double> other(ctx, 999);
    BOOST_CHECK_THROW(vex::inclusive_scan(vals, other), std::runtime_error);
}
