// vex::raw_pointer: the two CUDA cases of the reference's tests/vector_pointer.cpp (only the Boost.Test harness
// replaced), then a raw_pointer of a two-part vector, which throws, and a rotation through a pointer into the target,
// which reads the old values.
#include "testing.hpp"
#include <vexcl/vector.hpp>
#include <vexcl/vector_pointer.hpp>
#include <vexcl/element_index.hpp>
#include <vexcl/tagged_terminal.hpp>
#include <vexcl/temporary.hpp>
#include <vexcl/constants.hpp>
#include <vexcl/function.hpp>
#include <vexcl/vexcl.hpp>

BOOST_AUTO_TEST_CASE(nbody)
{
    const size_t n = 1024;

    std::vector<vex::command_queue> queue(1, ctx.queue(0));

    std::vector<double> X = random_vector<double>(n);

    vex::vector<double> x(queue, X);
    vex::vector<double> y(queue, n);

    VEX_FUNCTION(double, nbody, (size_t, n)(size_t, j)(double*, x),
            double sum = 0;
            for(size_t i = 0; i < n; ++i)
                if (i != j) sum += x[i];
                    return sum;
            );

    y = nbody(n, vex::element_index(), vex::raw_pointer(x));

    check_sample(y, [&](size_t idx, double v) {
            double sum = 0;
            for(size_t i = 0; i < n; ++i)
                if (i != idx) sum += X[i];
            BOOST_CHECK_CLOSE(v, sum, 1e-8);
            });
}

BOOST_AUTO_TEST_CASE(manual_stencil)
{
    const size_t n = 1024;

    std::vector<vex::command_queue> queue(1, ctx.queue(0));

    std::vector<double> X = random_vector<double>(n);

    vex::vector<double> x(queue, X);
    vex::vector<double> y(queue, n);

    VEX_CONSTANT(nil, 0);
    VEX_CONSTANT(one, 1);
    VEX_CONSTANT(two, 2);

    auto N = vex::tag<1>( x.size() );
    auto p = vex::raw_pointer(x);

    auto i     = vex::make_temp<1>( vex::element_index() );
    auto left  = vex::make_temp<2>( if_else(i > nil(), i - one(), i ) );
    auto right = vex::make_temp<3>( if_else(i + one() < N, i + one(), i ) );

    // Use pointer arithmetics
    y = *(p + i) * two() - *(p + left) - *(p + right);

    check_sample(y, [&](size_t idx, double v) {
            double xc = X[idx];
            double xl = X[idx > 0 ? idx - 1 : idx];
            double xr = X[idx + 1 < n ? idx + 1 : idx];
            BOOST_CHECK_CLOSE(v, 2 * xc - xr - xl, 1e-8);
            });

    // Same thing with index operators
    y = p[i] * two() - p[left] - p[right];

    check_sample(y, [&](size_t idx, double v) {
            double xc = X[idx];
            double xl = X[idx > 0 ? idx - 1 : idx];
            double xr = X[idx + 1 < n ? idx + 1 : idx];
            BOOST_CHECK_CLOSE(v, 2 * xc - xr - xl, 1e-8);
            });
}

// The reference refuses a pointer into a vector of several parts; with VEXCL_TEST_PARTS=1 the context has one part, and
// a vector over the context's queue duplicated stands in for a two-part vector.
BOOST_AUTO_TEST_CASE(raw_pointer_of_two_parts_throws)
{
    std::vector<vex::command_queue> two(2, ctx.queue(0));
    vex::vector<double> x(two, 1000);
    BOOST_CHECK_THROW(vex::raw_pointer(x), std::runtime_error);

    // a one-part pointer next to a two-part vector: refused before anything is launched
    std::vector<vex::command_queue> one(1, ctx.queue(0));
    vex::vector<double> z(one, 1000);
    z = 1;
    auto p = vex::raw_pointer(z);
    BOOST_CHECK_THROW(x = p[vex::element_index()], std::runtime_error);
}

// x = p[(i + 1) % n] with p = raw_pointer(x): every element reads the old x (the reference races here), through the
// interpreter, the generated kernel and a multi-expression.
BOOST_AUTO_TEST_CASE(rotation_through_aliased_pointer)
{
    const size_t n = 100003;
    std::vector<vex::command_queue> queue(1, ctx.queue(0));
    std::vector<double> X = random_vector<double>(n);
    vex::vector<double> x(queue, X);
    auto p = vex::raw_pointer(x);
    for (int round = 0; round < 3; ++round) {
        x = p[(vex::element_index() + 1) % n];
        std::rotate(X.begin(), X.begin() + 1, X.end());
        std::vector<double> got(n);
        vex::copy(x, got);
        BOOST_CHECK(got == X);
    }

    vex::vector<double> y(queue, n);
    y = 0;
    vex::tie(x, y) = std::make_tuple(p[(vex::element_index() + n - 1) % n], p[vex::element_index()] * 2);
    std::vector<double> gx(n), gy(n);
    vex::copy(x, gx); vex::copy(y, gy);
    for (size_t k = 0; k < n; ++k) {
        BOOST_CHECK_EQUAL(gx[k], X[(k + n - 1) % n]);
        BOOST_CHECK_EQUAL(gy[k], X[k] * 2);
    }
}

