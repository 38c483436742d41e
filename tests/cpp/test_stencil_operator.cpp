// VEX_STENCIL_OPERATOR through include/vexcl, bit for bit.  The bodies' device results are exactly defined (+, -, *,
// constants exact in T; NVRTC compiles them with --fmad=false), so each output is compared with the same operations
// done on the host, at lengths 1 to 257.  A 41-tap operator has halos longer than the neighbouring slice, so over two
// slices detail::stencil_halos pads them from the ends of the vector; its event-ordered exchange is tested only here.
#include "testing.hpp"

namespace {

// x[clamp(i + shift)]: the element k places from i, clamped at the ends of the vector
double clamped(const std::vector<double> &x, size_t i, long shift) {
    const long j = static_cast<long>(i) + shift, n = static_cast<long>(x.size());
    return x[static_cast<size_t>(j < 0 ? 0 : (j >= n ? n - 1 : j))];
}

// y = f(X) and y += 0.5 * f(X); `f` takes the accessor k -> X[k] and repeats the body's operations in order.
template <class Op, class F>
void run_operator_case(const Op &op, size_t n, F f) {
    const std::vector<double> host = random_vector<double>(n), init = random_vector<double>(n);
    vex::vector<double> X(ctx, host), Y(ctx, n);
    std::vector<double> back(n);
    auto want = [&](size_t i) { return f([&](long k) { return clamped(host, i, k); }); };
    Y = op(X);
    copy(Y, back);
    for (size_t i = 0; i < n; ++i) BOOST_CHECK(back[i] == want(i));
    copy(init, Y);
    Y += 0.5 * op(X);
    copy(Y, back);
    for (size_t i = 0; i < n; ++i) BOOST_CHECK(back[i] == init[i] + 0.5 * want(i));
}

} // namespace

BOOST_AUTO_TEST_CASE(second_difference_and_one_sided_operators)
{
    VEX_STENCIL_OPERATOR(second_difference, double, 3, 1, "return X[-1] - (T)2 * X[0] + X[1];", ctx);
    VEX_STENCIL_OPERATOR(forward, double, 3, 0, "return X[2] - (T)2 * X[1] + X[0];", ctx);
    VEX_STENCIL_OPERATOR(backward, double, 3, 2, "return (T)0.5 * (X[0] - X[-2]) + X[-1] * X[-1];", ctx);
    for (size_t n : {1u, 2u, 17u, 33u, 257u}) {
        run_operator_case(second_difference, n, [](auto X) { return X(-1) - 2.0 * X(0) + X(1); });
        run_operator_case(forward, n, [](auto X) { return X(2) - 2.0 * X(1) + X(0); });
        run_operator_case(backward, n, [](auto X) { return 0.5 * (X(0) - X(-2)) + X(-1) * X(-1); });
    }
}

BOOST_AUTO_TEST_CASE(wide_operator_with_halos_past_a_slice)
{
    // 20 elements either side: longer than the slices of 16 and 1 elements that two slices of n = 17 give
    VEX_STENCIL_OPERATOR(sum_squares, double, 41, 20,
                         "T s = (T)0;\nfor (int k = -CENTER; k <= RHALO; ++k) s = s + X[k] * X[k];\nreturn s;", ctx);
    for (size_t n : {1u, 2u, 17u, 33u, 257u})
        run_operator_case(sum_squares, n, [](auto X) { double s = 0; for (long k = -20; k <= 20; ++k) s = s + X(k) * X(k); return s; });
}
