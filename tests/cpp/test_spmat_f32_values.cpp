// vex::SpMat<double> with float-stored values (VEXB_FMT_VALUES_F32): every product must have the bits of the
// vex::SpMat<double> built from the values rounded to float, on one slice and on two (VEXCL_TEST_PARTS).
#include "testing.hpp"
#include <cstring>

static bool same_bits(const std::vector<double> &a, const std::vector<double> &b) {
    return a.size() == b.size() && std::memcmp(a.data(), b.data(), a.size() * sizeof(double)) == 0;
}

static std::vector<double> read(const vex::vector<double> &Y) {
    std::vector<double> h(Y.size());
    vex::copy(Y, h);
    return h;
}

static void check_format(int fmt, size_t n, size_t m, const std::vector<size_t> &row, const std::vector<size_t> &col,
                         const std::vector<double> &val)
{
    std::vector<double> rval(val.size());
    for (size_t j = 0; j < val.size(); ++j) rval[j] = static_cast<double>(static_cast<float>(val[j]));
    vex::SpMat<double> A(ctx, n, m, row.data(), col.data(), val.data(), fmt | VEXB_FMT_VALUES_F32);
    vex::SpMat<double> D(ctx, n, m, row.data(), col.data(), rval.data(), fmt);
    vex::SpMat<double> U(ctx, n, m, row.data(), col.data(), val.data(), fmt);
    BOOST_CHECK_EQUAL(A.info().loc.fmt, D.info().loc.fmt);
    BOOST_CHECK_EQUAL(A.info().loc.ell_width, D.info().loc.ell_width);

    std::vector<double> x = random_vector<double>(m);
    vex::vector<double> X(ctx, x), Ya(ctx, n), Yd(ctx, n), Yu(ctx, n), Zr(ctx, random_vector<double>(n));
    const vex::vector<double> &Z = n == m ? X : Zr;         // Y = X + A*X on square matrices

    Ya = A * X; Yd = D * X; Yu = U * X;
    BOOST_CHECK(same_bits(read(Ya), read(Yd)));
    BOOST_CHECK(!same_bits(read(Ya), read(Yu)));            // the flag is not ignored

    Ya -= 2 * (A * X); Yd -= 2 * (D * X);
    BOOST_CHECK(same_bits(read(Ya), read(Yd)));

    Ya = Z + A * X; Yd = Z + D * X;
    BOOST_CHECK(same_bits(read(Ya), read(Yd)));

    // inlined: the float-valued strip is not walked by the generated row loop, its product goes through a temporary
    Ya = Z + vex::make_inline(A * X); Yd = Z + vex::make_inline(D * X);
    BOOST_CHECK(same_bits(read(Ya), read(Yd)));
    BOOST_CHECK(!A.inline_strip(0));
}

BOOST_AUTO_TEST_CASE(float_values_random)
{
    const size_t n = 4096;
    for (int fmt : {VEXB_FMT_AUTO, VEXB_FMT_CSR, VEXB_FMT_HELL, VEXB_FMT_SELL}) {
        std::vector<size_t> row, col; std::vector<double> val;
        random_matrix(n, n, 16, row, col, val);
        check_format(fmt, n, n, row, col, val);
    }
}

BOOST_AUTO_TEST_CASE(float_values_poisson)
{
    const size_t g = 64, n = g * g;
    std::vector<size_t> row(1, 0), col; std::vector<double> val;
    std::vector<double> coef = random_vector<double>(5);
    for (size_t i = 0; i < n; ++i) {
        const long r = static_cast<long>(i);
        const long nb[5] = {r - static_cast<long>(g), r - 1, r, r + 1, r + static_cast<long>(g)};
        for (int k = 0; k < 5; ++k)
            if (nb[k] >= 0 && nb[k] < static_cast<long>(n)) { col.push_back(static_cast<size_t>(nb[k])); val.push_back(coef[k] + 1e-9 * static_cast<double>(i % 7)); }
        row.push_back(col.size());
    }
    check_format(VEXB_FMT_AUTO, n, n, row, col, val);
    check_format(VEXB_FMT_HELL, n, n, row, col, val);
}

BOOST_AUTO_TEST_CASE(float_values_rectangular)
{
    const size_t n = 1024, m = 3000;
    std::vector<size_t> row, col; std::vector<double> val;
    random_matrix(n, m, 16, row, col, val);
    check_format(VEXB_FMT_AUTO, n, m, row, col, val);
}
