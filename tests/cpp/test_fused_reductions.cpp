// Reductions of expressions with inlined sparse products and user functions (sum(f - A*x), the reference's counting
// sums): one launch per slice, and the bits of evaluating the expression into a temporary and reducing that, on one
// slice and on two (VEXCL_TEST_PARTS).
#include "testing.hpp"
#include <cstring>
#include <vexcl/sparse/matrix.hpp>

VEX_FUNCTION(size_t, greater_fn, (double, x)(double, y), return x > y;);
VEX_FUNCTION(double, times2, (double, x), return x * 2;);

template <class T> static bool same_bits(const T &a, const T &b) { return std::memcmp(&a, &b, sizeof(T)) == 0; }

static uint64_t launches() { uint64_t n = 0; vexb_launch_count(&n); return n; }

// Row i of a 5-point-like band that stays inside the slice of row i, so the strips have no halo and inline.
static void block_band(size_t n, const std::vector<size_t> &part, std::vector<size_t> &row, std::vector<size_t> &col,
                       std::vector<double> &val) {
    const std::vector<double> coef = random_vector<double>(5);
    const long off[5] = {-300, -1, 0, 1, 300};
    row.assign(1, 0); col.clear(); val.clear();
    size_t d = 0;
    for (size_t i = 0; i < n; ++i) {
        while (i >= part[d + 1]) ++d;
        for (int k = 0; k < 5; ++k) {
            const long c = static_cast<long>(i) + off[k];
            if (c >= static_cast<long>(part[d]) && c < static_cast<long>(part[d + 1])) {
                col.push_back(static_cast<size_t>(c)); val.push_back(coef[k] * (1 + 1e-3 * static_cast<double>(i % 11)));
            }
        }
        row.push_back(col.size());
    }
}

BOOST_AUTO_TEST_CASE(residual_with_spmat_make_inline)
{
    const size_t n = 100003;
    const std::vector<size_t> part = vex::partition(n, ctx.queue());
    std::vector<size_t> row, col; std::vector<double> val;
    block_band(n, part, row, col, val);
    for (int fmt : {VEXB_FMT_CSR, VEXB_FMT_HELL}) {
        vex::SpMat<double> A(ctx, n, n, row.data(), col.data(), val.data(), fmt);
        BOOST_REQUIRE(A.inlinable());
        vex::vector<double> X(ctx, random_vector<double>(n)), F(ctx, random_vector<double>(n)), T(ctx, n);
        vex::Reductor<double, vex::SUM> sum(ctx);
        vex::Reductor<double, vex::SUM_Kahan> csum(ctx);
        vex::Reductor<double, vex::MIN_MAX> minmax(ctx);

        uint64_t l0 = launches();
        const double s = sum(F - vex::make_inline(A * X));
        BOOST_CHECK_EQUAL(launches() - l0, ctx.size());
        T = F - vex::make_inline(A * X);
        BOOST_CHECK(same_bits(s, sum(T)));

        const double c = csum(fabs(F - vex::make_inline(A * X)));
        T = fabs(F - vex::make_inline(A * X));
        BOOST_CHECK(same_bits(c, csum(T)));

        l0 = launches();
        const auto mm = minmax(F - vex::make_inline(A * X));
        BOOST_CHECK_EQUAL(launches() - l0, ctx.size());
        T = F - vex::make_inline(A * X);
        const auto mt = minmax(T);
        BOOST_CHECK(same_bits(mm.s[0], mt.s[0]) && same_bits(mm.s[1], mt.s[1]));

        // a residual and its norms in one pass
        vex::Reductor<double, vex::CombineReductors<vex::SUM, vex::SUM_Kahan, vex::MAX, vex::MIN, vex::SUM>> five(ctx);
        l0 = launches();
        const auto r5 = five(F - vex::make_inline(A * X));
        BOOST_CHECK_EQUAL(launches() - l0, ctx.size());
        T = F - vex::make_inline(A * X);
        const auto t5 = five(T);
        for (int k = 0; k < 5; ++k) BOOST_CHECK(same_bits(r5.s[k], t5.s[k]));
    }
}

BOOST_AUTO_TEST_CASE(residual_with_sparse_matrix)
{
    const size_t n = 65537;
    std::vector<vex::command_queue> q(1, ctx.queue(0));
    std::vector<size_t> row, col; std::vector<double> val;
    block_band(n, std::vector<size_t>{0, n}, row, col, val);
    const std::vector<int> ptr(row.begin(), row.end()), idx(col.begin(), col.end());
    vex::sparse::matrix<double> A(q, n, n, ptr, idx, val);
    vex::vector<double> X(q, random_vector<double>(n)), F(q, random_vector<double>(n)), T(q, n);
    vex::Reductor<double, vex::SUM> sum(q);
    const uint64_t l0 = launches();
    const double s = sum(F - A * X);
    BOOST_CHECK_EQUAL(launches() - l0, 1u);
    T = F - A * X;
    BOOST_CHECK(same_bits(s, sum(T)));
    const double s2 = sum((F - A * X) * (F - A * X));
    T = (F - A * X) * (F - A * X);
    BOOST_CHECK(same_bits(s2, sum(T)));
}

// vector_arithmetics.cpp:113-145 (user_defined_functions)
BOOST_AUTO_TEST_CASE(counting_sums)
{
    const size_t N = 1 << 20;
    std::vector<double> xh = random_vector<double>(N), yh = random_vector<double>(N);
    vex::vector<double> x(ctx, xh), y(ctx, yh);
    vex::vector<double> td(ctx, N);
    vex::Reductor<size_t, vex::SUM> count(ctx);
    vex::Reductor<double, vex::SUM> sum(ctx);
    size_t want = 0;
    for (size_t i = 0; i < N; ++i) want += xh[i] > yh[i];

    uint64_t l0 = launches();
    const size_t c = count(greater_fn(x, y));
    BOOST_CHECK_EQUAL(launches() - l0, ctx.size());
    BOOST_CHECK_EQUAL(c, want);
    BOOST_CHECK_EQUAL(count(greater_fn(x, y)) + count(greater_fn(y, x)), N);          // random doubles: no ties

    l0 = launches();
    const double s = sum(times2(x));
    BOOST_CHECK_EQUAL(launches() - l0, ctx.size());
    td = times2(x);
    BOOST_CHECK(same_bits(s, sum(td)));

    x = 1; y = 2;
    BOOST_CHECK_EQUAL(count(greater_fn(x, y)), 0u);
    BOOST_CHECK_EQUAL(count(greater_fn(y, x)), N);
    BOOST_CHECK_EQUAL(sum(times2(x)), 2.0 * N);
}
