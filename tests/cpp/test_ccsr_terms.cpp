// vex::SpMatCCSR products as expression terminals (the reference's ccsr_product, spmat/ccsr.hpp:88-270): `sin(A*X)`,
// `X * (A*X)`, `sum(X * (A*X))`, make_inline(A*X), compound assignments, user functions and if_else, on the matrix of the
// reference's ccsr_vector_product test (tests/spmv.cpp:148-231), one slice, against host loops.  Neither side contracts
// a*b+c, so every value without a math function is compared exactly; sums and sin() within a tolerance.
#include <algorithm>
#include "testing.hpp"
#include <vexcl/spmat/ccsr.hpp>

VEX_FUNCTION(double, sq, (double, a), return a * a;);

namespace {
struct poisson32 {
    const size_t n = 32, N = n * n * n;
    std::vector<size_t> idx, row = {0, 1, 8};
    std::vector<int> col;
    std::vector<double> val;
    std::vector<double> x;
    poisson32() {
        const double h2i = (n - 1) * (n - 1);
        const int nn = static_cast<int>(n * n), n1 = static_cast<int>(n);
        col = {0, -nn, -n1, -1, 0, 1, n1, nn};
        val = {1, -h2i, -h2i, -h2i, 6 * h2i, -h2i, -h2i, -h2i};
        for (size_t k = 0; k < n; k++)
            for (size_t j = 0; j < n; j++)
                for (size_t i = 0; i < n; i++)
                    idx.push_back(i == 0 || i == n - 1 || j == 0 || j == n - 1 || k == 0 || k == n - 1 ? 0 : 1);
        x = random_vector<double>(N);
    }
    double row_sum(size_t ii) const {
        double sum = 0;
        for (size_t j = row[idx[ii]]; j < row[idx[ii] + 1]; j++) sum = sum + val[j] * x[ii + col[j]];
        return sum;
    }
};

uint64_t launches() { uint64_t l = 0; vexb_launch_count(&l); return l; }
}

BOOST_AUTO_TEST_CASE(ccsr_terminal_spellings)
{
    poisson32 p;
    std::vector<vex::command_queue> queue(1, ctx.queue(0));
    vex::SpMatCCSR<double, int> A(queue[0], p.N, p.row.size() - 1, p.idx.data(), p.row.data(), p.col.data(), p.val.data());
    vex::vector<double> X(queue, p.x), Y(queue, p.N);

    Y = sin(A * X);
    check_sample(Y, [&](size_t i, double a) { BOOST_CHECK_CLOSE(a, std::sin(p.row_sum(i)), 1e-10); });
    Y = X * (A * X);
    check_sample(Y, [&](size_t i, double a) { BOOST_CHECK_EQUAL(a, p.x[i] * p.row_sum(i)); });
    Y = (A * X) * X;
    check_sample(Y, [&](size_t i, double a) { BOOST_CHECK_EQUAL(a, p.row_sum(i) * p.x[i]); });
    Y = X * (2 * (A * X));                                              // the scale goes into the expression
    check_sample(Y, [&](size_t i, double a) { BOOST_CHECK_EQUAL(a, p.x[i] * (2 * p.row_sum(i))); });
    Y = vex::make_inline(A * X) * 2.0 + X;
    check_sample(Y, [&](size_t i, double a) { BOOST_CHECK_EQUAL(a, p.row_sum(i) * 2.0 + p.x[i]); });
    Y = sq(A * X);
    check_sample(Y, [&](size_t i, double a) { BOOST_CHECK_EQUAL(a, p.row_sum(i) * p.row_sum(i)); });
    Y = vex::if_else(A * X > 0, X, A * X);
    check_sample(Y, [&](size_t i, double a) { const double s = p.row_sum(i); BOOST_CHECK_EQUAL(a, s > 0 ? p.x[i] : s); });
    Y = X;
    Y *= A * X;
    check_sample(Y, [&](size_t i, double a) { BOOST_CHECK_EQUAL(a, p.x[i] * p.row_sum(i)); });
    Y /= A * X;
    check_sample(Y, [&](size_t i, double a) { BOOST_CHECK_EQUAL(a, (p.x[i] * p.row_sum(i)) / p.row_sum(i)); });
    // the additive spellings keep the hand-written kernels, with the same values
    Y = A * X;
    check_sample(Y, [&](size_t i, double a) { BOOST_CHECK_EQUAL(a, p.row_sum(i)); });
    Y = X + A * X;
    check_sample(Y, [&](size_t i, double a) { BOOST_CHECK_EQUAL(a, p.x[i] + p.row_sum(i)); });
    Y -= 0.5 * (A * X);
    check_sample(Y, [&](size_t i, double a) { BOOST_CHECK_EQUAL(a, (p.x[i] + p.row_sum(i)) + (-0.5 * p.row_sum(i))); });
}

BOOST_AUTO_TEST_CASE(ccsr_terminal_reductions)
{
    poisson32 p;
    std::vector<vex::command_queue> queue(1, ctx.queue(0));
    vex::SpMatCCSR<double, int> A(queue[0], p.N, p.row.size() - 1, p.idx.data(), p.row.data(), p.col.data(), p.val.data());
    vex::vector<double> X(queue, p.x);
    vex::Reductor<double, vex::SUM> sum(queue);
    vex::Reductor<double, vex::MIN_MAX> minmax(queue);
    vex::Reductor<double, vex::CombineReductors<vex::SUM, vex::MAX>> summax(queue);
    double e = 0, s = 0, lo = p.row_sum(0), hi = lo;
    for (size_t i = 0; i < p.N; ++i) {
        const double r = p.row_sum(i);
        e += p.x[i] * r; s += r; lo = std::min(lo, r); hi = std::max(hi, r);
    }
    BOOST_CHECK_CLOSE(sum(X * (A * X)), e, 1e-8);                       // the energy norm of the reference's examples
    BOOST_CHECK_CLOSE(sum(A * X), s, 1e-8);
    auto m = minmax(A * X);
    BOOST_CHECK_EQUAL(m.s[0], lo);
    BOOST_CHECK_EQUAL(m.s[1], hi);
    auto c = summax(vex::make_inline(A * X));
    BOOST_CHECK_CLOSE(c.s[0], s, 1e-8);
    BOOST_CHECK_EQUAL(c.s[1], hi);
}

BOOST_AUTO_TEST_CASE(ccsr_terminal_launches_and_aliasing)
{
    poisson32 p;
    std::vector<vex::command_queue> queue(1, ctx.queue(0));
    vex::SpMatCCSR<double, int> A(queue[0], p.N, p.row.size() - 1, p.idx.data(), p.row.data(), p.col.data(), p.val.data());
    vex::vector<double> X(queue, p.x), Y(queue, p.N);
    vex::Reductor<double, vex::SUM> sum(queue);
    Y = X * (A * X);                                                    // warm: the kernels are generated at first use
    sum(X * (A * X));
    uint64_t l0 = launches();
    Y = X * (A * X);
    BOOST_CHECK_EQUAL(launches() - l0, 1u);
    l0 = launches();
    sum(X * (A * X));
    BOOST_CHECK_EQUAL(launches() - l0, 1u);
    // x as the target: the product goes to a temporary first
    vex::vector<double> Z(queue, p.x);
    Z = X * (A * Z);
    check_sample(Z, [&](size_t i, double a) { BOOST_CHECK_EQUAL(a, p.x[i] * p.row_sum(i)); });
    // one slice only, as in the reference
    if (ctx.size() > 1) {
        vex::vector<double> X2(ctx, p.x), Y2(ctx, p.N);
        BOOST_CHECK_THROW(Y2 = sin(A * X2), std::runtime_error);
    }
}
