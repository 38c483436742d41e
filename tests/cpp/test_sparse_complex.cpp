// Complex values of vex::sparse matrices: the body of the reference's examples/complex_spmv.cpp main() against
// include/vexcl/sparse, for csr, ell and matrix, then random complex matrices in both precisions with `Y = A * X`,
// `Y += A * X` and `Y -= A * X`.
#include "testing.hpp"
#include <complex>
#include <sstream>
#include <vexcl/sparse/matrix.hpp>
#include <vexcl/sparse/distributed.hpp>

template <class T> constexpr double close_pct() { return std::is_same<T, double>::value ? 1e-8 : 1e-3; }

// sum over the entries of row i in storage order, the arithmetic of the example's spmv_ops_impl
template <class T>
static std::complex<T> row_product(const std::vector<int> &ptr, const std::vector<int> &col,
                                   const std::vector<std::complex<T>> &val, const std::vector<std::complex<T>> &x, size_t i) {
    T re = 0, im = 0;
    for (int j = ptr[i]; j < ptr[i + 1]; j++) {
        const T a = val[j].real(), b = val[j].imag(), xr = x[col[j]].real(), xi = x[col[j]].imag();
        re += a * xr - b * xi;
        im += a * xi + b * xr;
    }
    return std::complex<T>(re, im);
}

// examples/complex_spmv.cpp main(), with the matrix class as a parameter and the printed Y checked
template <class M>
static void example_case()
{
    vex::Context ctx1(vex::Filter::Env && vex::Filter::Count(1));
    std::cout << ctx1 << std::endl;

    // 4x4 diagonal matrix in CSR format:
    std::vector<int> ptr = {0,1,2,3,4};
    std::vector<int> col = {0,1,2,3};
    std::vector<std::complex<double>> val = {
        {1.0, 1.0}, {2.0, 2.0}, {3.0, 3.0}, {4.0, 4.0}};

    // complex vector:
    std::vector<std::complex<double>> x = {
        {1.0, 1.0}, {1.0, 1.0}, {1.0, 1.0}, {1.0, 1.0}};

    // Device-side matrix and vectors:
    M A(ctx1, 4, 4, ptr, col, val);
    vex::vector<std::complex<double>> X(ctx1, x);
    vex::vector<std::complex<double>> Y(ctx1, 4);

    Y = A * X;

    std::cout << Y << std::endl;

    BOOST_CHECK_EQUAL(A.rows(), 4u);
    BOOST_CHECK_EQUAL(A.nonzeros(), 4u);
    for (int k = 0; k < 4; ++k) {                          // (k+1)(1+i) * (1+i) = 2(k+1) i, exactly
        std::complex<double> y = Y[k];
        BOOST_CHECK(y == std::complex<double>(0.0, 2.0 * (k + 1)));
    }
    std::ostringstream s;
    s << Y;
    BOOST_CHECK(s.str().find("(0,8)") != std::string::npos);
}

template <class M, class T>
static void random_case()
{
    typedef std::complex<T> Z;
    const size_t n = 1024, m = 777;
    std::vector<vex::command_queue> q(1, ctx.queue(0));
    std::vector<int> ptr, col; std::vector<T> scalars;
    random_matrix(n, m, 16, ptr, col, scalars);
    std::vector<Z> val(col.size());
    for (auto &a : val) a = Z(generator<T>::get() - T(0.5), generator<T>::get() - T(0.5));
    std::vector<Z> x(m), z(n);
    for (auto &v : x) v = Z(generator<T>::get(), generator<T>::get());
    for (auto &v : z) v = Z(generator<T>::get(), generator<T>::get());

    M A(q, n, m, ptr, col, val);
    BOOST_CHECK_EQUAL(A.cols(), m);
    vex::vector<Z> X(q, x), Y(q, n), Z_(q, z);

    Y = A * X;
    check_sample(Y, [&](size_t i, Z y) {
        const Z sum = row_product(ptr, col, val, x, i);
        BOOST_CHECK_CLOSE(y.real(), sum.real(), close_pct<T>());
        BOOST_CHECK_CLOSE(y.imag(), sum.imag(), close_pct<T>());
    });

    Z_ += A * X;                                          // z + s
    check_sample(Z_, [&](size_t i, Z y) {
        const Z sum = row_product(ptr, col, val, x, i);
        BOOST_CHECK_CLOSE(y.real(), z[i].real() + sum.real(), close_pct<T>());
        BOOST_CHECK_CLOSE(y.imag(), z[i].imag() + sum.imag(), close_pct<T>());
    });
    Z_ -= A * X;
    Z_ -= A * X;                                          // (z + s) - s - s
    check_sample(Z_, [&](size_t i, Z y) {
        const Z sum = row_product(ptr, col, val, x, i);
        const Z want = (z[i] + sum) - sum - sum;
        BOOST_CHECK_SMALL(std::abs(y - want), 1e-4 * (std::abs(z[i]) + 3 * std::abs(sum) + 1));
    });

    // the vectors' bytes are (re, im) per element, in order (vex::copy and element reads agree)
    std::vector<Z> back(n);
    vex::copy(Z_, back);
    for (size_t i = 0; i < n; i += 101) { Z e = Z_[i]; BOOST_CHECK(e == back[i]); }
}

BOOST_AUTO_TEST_CASE(complex_spmv_example)
{
    example_case<vex::sparse::matrix<std::complex<double>>>();
    example_case<vex::sparse::csr<std::complex<double>>>();
    example_case<vex::sparse::ell<std::complex<double>>>();
}

template <class T>
static void all_formats() {
    random_case<vex::sparse::csr<std::complex<T>>, T>();
    random_case<vex::sparse::ell<std::complex<T>>, T>();
    random_case<vex::sparse::matrix<std::complex<T>>, T>();
}

BOOST_AUTO_TEST_CASE(complex_double) { all_formats<double>(); }
BOOST_AUTO_TEST_CASE(complex_float)  { all_formats<float>(); }

BOOST_AUTO_TEST_CASE(complex_matrix_needs_one_device)
{
    // like the scalar and block classes: a context of two queues is refused at construction
    std::vector<int> ptr = {0, 1}, col = {0};
    std::vector<std::complex<double>> val(1, std::complex<double>(1, 1));
    std::vector<vex::command_queue> q2(2, ctx.queue(0));
    BOOST_CHECK_THROW(vex::sparse::matrix<std::complex<double>> A(q2, 1, 1, ptr, col, val), std::exception);
}
