// User functions with dependencies and preambles, and per-device program headers, through include/vexcl.  The first
// four cases are the reference's (tests/vector_arithmetics.cpp:131-236) as written there; the rest extend them.  Bodies
// use +, -, * only where a result is compared exactly: NVRTC compiles them with --fmad=false, and the host repeats the
// same operations in the same order.
#include "testing.hpp"

BOOST_AUTO_TEST_CASE(user_defined_functions_same_signature)
{
    const size_t N = 1024;
    vex::vector<double> x(ctx, N);

    x = 1;

    VEX_FUNCTION(double, times2, (double, x), return x * 2;);
    VEX_FUNCTION(double, times4, (double, x), return x * 4;);

    vex::Reductor<size_t,vex::SUM> sum(ctx);

    BOOST_CHECK( sum( times2(x) ) == 2 * N );
    BOOST_CHECK( sum( times4(x) ) == 4 * N );
}

BOOST_AUTO_TEST_CASE(nested_functions)
{
    const size_t N = 1024;

    VEX_FUNCTION(int, f, (int, x), return 2 * x;);
    VEX_FUNCTION(int, g, (int, x), return 3 * x;);

    vex::vector<int> x(ctx, N);

    x = 1;
    x = f(f(x));
    check_sample(x, [](size_t, int a) { BOOST_CHECK(a == 4); });

    x = 1;
    x = g(f(x));
    check_sample(x, [](size_t, int a) { BOOST_CHECK(a == 6); });
}

BOOST_AUTO_TEST_CASE(custom_header)
{
    const size_t n = 1024;

    vex::vector<int> x(ctx, n);

    vex::push_program_header(ctx, "#define THE_ANSWER 42\n");

    VEX_FUNCTION(int, answer, (int, x), return x * THE_ANSWER;);

    x = answer(1);

    check_sample(x, [](size_t, int a) {
            BOOST_CHECK(a == 42);
            });

    vex::pop_program_header(ctx);
}

// Have to define these outside of the following test case scope.
// In Visual C++ is not types defined in enclosing function scope
// are not able to refeence each other.
VEX_FUNCTION(double, sin2, (double, x), return pow(sin(x), 2.0););
VEX_FUNCTION(double, cos2, (double, x), return pow(cos(x), 2.0););

BOOST_AUTO_TEST_CASE(function_with_preamble)
{
    const size_t n = 1024;

    vex::vector<double> x(ctx, random_vector<double>(n));
    vex::vector<double> y(ctx, n);

    VEX_FUNCTION_D(double, one, (double, x), (sin2)(cos2),
            return sin2(x) + cos2(x);
            );

    y = one(x);

    check_sample(y, [](size_t, double a) {
            BOOST_CHECK_CLOSE(a, 1.0, 1e-8);
            });
}

// ---- beyond the reference's cases -------------------------------------------------------------------------------------
namespace {
std::vector<double> read(const vex::vector<double> &v) { std::vector<double> h(v.size()); vex::copy(v, h); return h; }
}

VEX_FUNCTION(double, step1, (double, x), return x + 1;);
VEX_FUNCTION_D(double, step2, (double, x), (step1), return step1(x) * 2;);
VEX_FUNCTION_SD(double, step3, (double, x), (step2), "return step2(x) - 3;");
VEX_FUNCTION(double, sq, (double, x), return x * x;);

BOOST_AUTO_TEST_CASE(three_level_dependency_chain)
{
    const size_t n = 1000;
    const std::vector<double> h = random_vector<double>(n);
    vex::vector<double> x(ctx, h), y(ctx, n);
    y = step3(x);
    const std::vector<double> got = read(y);
    for (size_t i = 0; i < n; ++i) BOOST_CHECK(got[i] == (h[i] + 1) * 2 - 3);
}

BOOST_AUTO_TEST_CASE(dependency_also_called_directly)
{
    const size_t n = 1000;
    const std::vector<double> h = random_vector<double>(n);
    vex::vector<double> x(ctx, h), y(ctx, n);
    y = step1(x) * step2(x) + step3(x);                 // step1 and step2 both as name_<id> and under their plain names
    const std::vector<double> got = read(y);
    for (size_t i = 0; i < n; ++i) BOOST_CHECK(got[i] == (h[i] + 1) * ((h[i] + 1) * 2) + ((h[i] + 1) * 2 - 3));
}

BOOST_AUTO_TEST_CASE(dependency_shared_by_two_functions)
{
    VEX_FUNCTION_D(double, twice_sq, (double, x), (sq), return 2 * sq(x););
    VEX_FUNCTION_DS(double, sq_plus, (double, x)(double, y), (sq), "return sq(x) + y;");
    const size_t n = 1000;
    const std::vector<double> h = random_vector<double>(n), g = random_vector<double>(n);
    vex::vector<double> x(ctx, h), z(ctx, g), y(ctx, n);
    y = twice_sq(x) - sq_plus(x, z);
    const std::vector<double> got = read(y);
    for (size_t i = 0; i < n; ++i) BOOST_CHECK(got[i] == 2 * (h[i] * h[i]) - (h[i] * h[i] + g[i]));
}

BOOST_AUTO_TEST_CASE(v1_function_with_preamble)
{
    // the reference's example (function.hpp:94-100): OpenCL-style helpers, without __device__, in the preamble
    VEX_FUNCTION_V1_WITH_PREAMBLE(one, double(double),
            "double sin2(double x) { return pow(sin(x), 2.0); }\n"
            "double cos2(double x) { return pow(cos(x), 2.0); }\n",
            "return sin2(prm1) + cos2(prm1);"
            );
    VEX_FUNCTION_V1_TYPE(cube, double(double), "", VEX_STRINGIZE_SOURCE(return prm1 * prm1 * prm1;));
    const vex_function_cube cube;
    const size_t n = 1024;
    const std::vector<double> h = random_vector<double>(n);
    vex::vector<double> x(ctx, h), y(ctx, n);
    y = one(x);
    check_sample(y, [](size_t, double a) { BOOST_CHECK_CLOSE(a, 1.0, 1e-8); });
    y = cube(x);
    const std::vector<double> got = read(y);
    for (size_t i = 0; i < n; ++i) BOOST_CHECK(got[i] == h[i] * h[i] * h[i]);
}

VEX_FUNCTION(double, scaled, (double, x), return x * SCALE;);

BOOST_AUTO_TEST_CASE(header_in_reduction_multiexpression_and_stencil_operator)
{
    const size_t n = 4099;
    const std::vector<double> h = random_vector<double>(n), g = random_vector<double>(n);
    vex::vector<double> x(ctx, h), z(ctx, g), a(ctx, n), b(ctx, n), t(ctx, n);
    vex::scoped_program_header header(ctx, "#define SCALE 3\n");
    BOOST_CHECK(vex::get_program_header(ctx.queue(0)) == "#define SCALE 3\n");

    vex::Reductor<double, vex::SUM> sum(ctx);
    t = x * 3.0;                                        // the reduction has the bits of the same expression on a temporary
    BOOST_CHECK(sum(scaled(x)) == sum(t));

    vex::tie(a, b) = std::make_tuple(scaled(x), scaled(z) + x);
    const std::vector<double> ga = read(a), gb = read(b);
    for (size_t i = 0; i < n; ++i) BOOST_CHECK(ga[i] == h[i] * 3 && gb[i] == g[i] * 3 + h[i]);

    VEX_STENCIL_OPERATOR(scaled_diff, double, 3, 1, "return SCALE * X[0] - X[1];", ctx);
    a = scaled_diff(x);
    const std::vector<double> gs = read(a);
    for (size_t i = 0; i < n; ++i) BOOST_CHECK(gs[i] == 3 * h[i] - h[i + 1 < n ? i + 1 : n - 1]);
}

VEX_FUNCTION(int, times_value, (int, x), return x * THE_VALUE;);

BOOST_AUTO_TEST_CASE(header_push_pop_push)
{
    const size_t n = 1024;
    vex::vector<int> x(ctx, n), y(ctx, n);
    x = vex::element_index();
    auto check_times = [&](int k) {
        std::vector<int> got(n);
        vex::copy(y, got);
        for (size_t i = 0; i < n; ++i) BOOST_CHECK(got[i] == static_cast<int>(i) * k);
    };
    vex::push_program_header(ctx, "#define THE_VALUE 2\n");
    y = times_value(x);
    check_times(2);
    vex::push_program_header(ctx, "#define THE_VALUE 5\n");       // a push replaces the header
    y = times_value(x);
    check_times(5);
    vex::pop_program_header(ctx);                                  // and a pop restores the previous one
    y = times_value(x);
    check_times(2);
    vex::pop_program_header(ctx);
    BOOST_CHECK(vex::get_program_header(ctx.queue(0)).empty());
    {
        vex::scoped_program_header header(ctx, "#define THE_VALUE 7");   // no trailing newline
        y = times_value(x);
        check_times(7);
    }
    BOOST_CHECK(vex::get_program_header(ctx.queue(0)).empty());
    BOOST_CHECK_THROW(vex::pop_program_header(ctx), vex::backend::error);
}
