// vex::make_temp: the five cases of the reference's tests/temporary.cpp (only the Boost.Test harness replaced), then
// temporaries of sparse products, an explicit type that differs from the deduced one, and one tag over two expressions.
#include "testing.hpp"
#include <vexcl/vector.hpp>
#include <vexcl/multivector.hpp>
#include <vexcl/temporary.hpp>
#include <vexcl/reductor.hpp>
#include <vexcl/function.hpp>

BOOST_AUTO_TEST_CASE(temporary)
{
    const size_t n = 1024;

    vex::vector<double> x(ctx, random_vector<double>(n));
    vex::vector<double> y(ctx, n);

    VEX_FUNCTION(double, sqr, (double, x), return x * x;);

    {
        // Deduce temporary type
        auto s = vex::make_temp<1>( sqr(x) + 25 );
        y = s * (x + s);

        check_sample(y, [&](size_t idx, double v) {
                double X = x[idx];
                double S = X * X + 25;
                BOOST_CHECK_CLOSE(v, S * (X + S), 1e-8);
                });
    }

    {
        // Provide temporary type
        auto s = vex::make_temp<1, double>( sqr(x) + 25 );
        y = s * (x + s);

        check_sample(y, [&](size_t idx, double v) {
                double X = x[idx];
                double S = X * X + 25;
                BOOST_CHECK_CLOSE(v, S * (X + S), 1e-8);
                });
    }
}

BOOST_AUTO_TEST_CASE(nested_temporary)
{
    const size_t n = 1024;

    vex::vector<double> x(ctx, random_vector<double>(n));
    vex::vector<double> y(ctx, n);

    auto t1 = vex::make_temp<1>( log(x) );
    auto t2 = vex::make_temp<2>( t1 + sin(x) );

    y = t1 * t2;

    check_sample(y, [&](size_t idx, double v) {
            double X = x[idx];
            double T1 = log(X);
            double T2 = T1 + sin(X);
            BOOST_CHECK_CLOSE(v, T1 * T2, 1e-8);
            });
}

BOOST_AUTO_TEST_CASE(reduce_temporary)
{
    const size_t n = 1024;

    vex::vector<double> x(ctx, random_vector<double>(n));

    auto t1 = vex::make_temp<1>( pow(sin(x), 2) );
    auto t2 = vex::make_temp<2>( pow(cos(x), 2) );

    vex::Reductor<double, vex::SUM> sum(ctx);

    BOOST_CHECK_CLOSE(sum(10 * (t1 + t2)), 10.0 * n, 1e-6);
}

BOOST_AUTO_TEST_CASE(multiexpression_temporary)
{
    typedef std::array<double, 2> elem_t;
    const size_t n = 1024;

    vex::vector<double> x(ctx, random_vector<double>(n));

    vex::multivector<double, 2> y(ctx,n);

    auto tmp = vex::make_temp<1>( sin(x) );

    y = std::tie(tmp, sqrt(1 - tmp * tmp));

    check_sample(y, [&](size_t idx, elem_t v){
            double X = x[idx];
            BOOST_CHECK_CLOSE(v[0], sin(X), 1e-8);
            BOOST_CHECK_CLOSE(v[1], cos(X), 1e-8);
            });
}

BOOST_AUTO_TEST_CASE(multivector_temporary)
{
    typedef std::array<double, 2> elem_t;
    const size_t n = 1024;

    vex::multivector<double, 2> x(ctx, random_vector<double>(2 * n));
    vex::multivector<double, 2> y(ctx,n);

    auto tmp = vex::make_temp<1, double>( tan(x) );

    y = tmp * tmp;

    check_sample(y, [&](size_t idx, elem_t v){
            elem_t X = x[idx];

            BOOST_CHECK_CLOSE(v[0], pow(tan(X[0]), 2.0), 1e-8);
            BOOST_CHECK_CLOSE(v[1], pow(tan(X[1]), 2.0), 1e-8);
            });
}

// ---- beyond the reference's file ----------------------------------------------------------------------------------

// make_temp<1, float> on double operands: the value is rounded to float once, every use reads that float
BOOST_AUTO_TEST_CASE(explicit_type_differs_from_deduced)
{
    const size_t n = 1024;
    vex::vector<double> x(ctx, random_vector<double>(n)), y(ctx, n);
    auto t = vex::make_temp<1, float>(x * 3 + 1);
    static_assert(std::is_same<decltype(t)::value_type, float>::value, "make_temp<Tag, T> has value type T");
    y = t * x;                                      // float * double: in double, as written out
    check_sample(y, [&](size_t i, double v) {
        const double X = x[i];
        BOOST_CHECK_EQUAL(v, static_cast<double>(static_cast<float>(X * 3 + 1)) * X);
    });
}

// y = t * t + t with t = A*x: in one launch when the product is inlined, with the bits of "product into a vector first"
BOOST_AUTO_TEST_CASE(temporary_of_inlined_products)
{
    const size_t n = 4096;
    std::vector<size_t> row, col; std::vector<double> val;
    random_matrix(n, n, 16, row, col, val);
    vex::SpMat<double> A(ctx, n, n, row.data(), col.data(), val.data());
    vex::vector<double> x(ctx, random_vector<double>(n)), y(ctx, n), z(ctx, n), w(ctx, n);
    auto t = vex::make_temp<1>(vex::make_inline(A * x));
    y = t * t + t;
    z = A * x;
    w = z * z + z;
    check_sample(y, w, [&](size_t, double a, double b) { BOOST_CHECK_EQUAL(a, b); });

    // SpMatCCSR products: one slice, as in the reference
    std::vector<vex::command_queue> q1(1, ctx.queue(0));
    const size_t m = 1000;
    std::vector<size_t> idx(m), crow = {0, 1, 4};
    std::vector<int> ccol = {0, -1, 0, 1};
    std::vector<double> cval = {1, -1, 2, -1};
    for (size_t i = 0; i < m; ++i) idx[i] = (i == 0 || i == m - 1) ? 0 : 1;
    vex::SpMatCCSR<double, int> C(q1[0], m, 2, idx.data(), crow.data(), ccol.data(), cval.data());
    vex::vector<double> X(q1, random_vector<double>(m)), Y(q1, m), Z(q1, m), W(q1, m);
    auto c = vex::make_temp<2>(C * X);
    Y = c * X + sin(c);
    Z = C * X;
    W = Z * X + sin(Z);
    check_sample(Y, W, [&](size_t, double a, double b) { BOOST_CHECK_EQUAL(a, b); });
}

// One tag is one temporary: the same tag over another expression is refused before anything runs
BOOST_AUTO_TEST_CASE(one_tag_two_expressions)
{
    const size_t n = 1024;
    vex::vector<double> x(ctx, random_vector<double>(n)), y(ctx, n);
    auto a = vex::make_temp<1>(sin(x));
    auto b = vex::make_temp<1>(cos(x));
    BOOST_CHECK_THROW(y = a + b, vex::backend::error);
    auto a2 = vex::make_temp<1>(sin(x));            // the same program under the same tag: one temporary
    y = a * a2;
    check_sample(y, [&](size_t i, double v) { BOOST_CHECK_CLOSE(v, std::sin(x[i]) * std::sin(x[i]), 1e-8); });
}
