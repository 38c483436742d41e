// Sliced-ELL strips (what vex::SpMat and vex::sparse::matrix choose for uneven rows) in the places hybrid ELL already
// serves: a product inlined into an assignment kernel (one launch, a storage-order sweep), and SpMat * multivector in one
// pass over the matrix.  Values against the reference tests' host loops (tests/spmv.cpp:233-260, :262-307,
// tests/sparse_matrices.cpp:66-124); launches counted on one device slice, where the strip has no halo.
#include <array>
#include "testing.hpp"
#include <vexcl/sparse/matrix.hpp>

template <class I>
static double row_sum(const std::vector<I> &row, const std::vector<I> &col, const std::vector<double> &val, const double *x, size_t i) {
    double sum = 0;
    for (size_t j = row[i]; j < static_cast<size_t>(row[i + 1]); j++) sum += val[j] * x[col[j]];
    return sum;
}

static uint64_t launches() { uint64_t l = 0; vexb_launch_count(&l); return l; }

BOOST_AUTO_TEST_CASE(product_in_assignment_is_one_launch)
{
    const size_t n = 4096;
    std::vector<vex::command_queue> queue(1, ctx.queue(0));
    std::vector<size_t> row, col; std::vector<double> val;
    random_matrix(n, n, 16, row, col, val);
    std::vector<double> x = random_vector<double>(n);
    vex::SpMat<double> A(queue, n, n, row.data(), col.data(), val.data());
    BOOST_REQUIRE(A.info().loc.fmt == VEXB_FMT_SELL);
    BOOST_CHECK(A.sweep_strip(0) != nullptr && A.inline_strip(0) == nullptr);
    vex::vector<double> X(queue, x), Y(queue, n);
    Y = X + A * X;                                                      // warm: the kernels are generated at first use
    Y -= 2 * (A * X);
    uint64_t l0 = launches();
    Y = X + A * X;
    BOOST_CHECK_EQUAL(launches() - l0, 1u);
    check_sample(Y, [&](size_t idx, double a) { BOOST_CHECK_CLOSE(a, x[idx] + row_sum(row, col, val, x.data(), idx), 1e-8); });
    l0 = launches();
    Y -= 2 * (A * X);
    BOOST_CHECK_EQUAL(launches() - l0, 1u);
    check_sample(Y, [&](size_t idx, double a) { BOOST_CHECK_CLOSE(a, x[idx] - row_sum(row, col, val, x.data(), idx), 1e-6); });
}

BOOST_AUTO_TEST_CASE(product_in_assignment_on_every_part)              // coupled parts fall back to the product kernels
{
    const size_t n = 4096;
    std::vector<size_t> row, col; std::vector<double> val;
    random_matrix(n, n, 16, row, col, val);
    std::vector<double> x = random_vector<double>(n);
    vex::SpMat<double> A(ctx, n, n, row.data(), col.data(), val.data());
    vex::vector<double> X(ctx, x), Y(ctx, n);
    Y = X + A * X;
    check_sample(Y, [&](size_t idx, double a) { BOOST_CHECK_CLOSE(a, x[idx] + row_sum(row, col, val, x.data(), idx), 1e-8); });
    Y -= 2 * (A * X);
    check_sample(Y, [&](size_t idx, double a) { BOOST_CHECK_CLOSE(a, x[idx] - row_sum(row, col, val, x.data(), idx), 1e-6); });
}

BOOST_AUTO_TEST_CASE(reduction_keeps_its_path)                          // tests/spmv.cpp:252-259
{
    const size_t n = 4096;
    std::vector<vex::command_queue> queue(1, ctx.queue(0));
    std::vector<size_t> row, col; std::vector<double> val;
    random_matrix(n, n, 16, row, col, val);
    std::vector<double> x = random_vector<double>(n), f(n);
    for (size_t i = 0; i < n; ++i) f[i] = row_sum(row, col, val, x.data(), i) + 0.25;
    vex::SpMat<double> A(queue, n, n, row.data(), col.data(), val.data());
    vex::vector<double> X(queue, x), F(queue, f);
    vex::Reductor<double, vex::SUM> sum(queue);
    const double eps = sum(fabs(F - vex::make_inline(A * X)));
    BOOST_CHECK_CLOSE(eps, 0.25 * n, 1e-8);
}

BOOST_AUTO_TEST_CASE(sparse_matrix_in_an_expression)
{
    const size_t n = 4096;
    std::vector<vex::command_queue> queue(1, ctx.queue(0));
    std::vector<int> row, col; std::vector<double> val;
    random_matrix(n, n, 16, row, col, val);
    std::vector<double> x = random_vector<double>(n);
    vex::sparse::matrix<double> A(queue, n, n, row, col, val);
    BOOST_CHECK(A.sweep_strip(0) != nullptr);
    vex::vector<double> X(queue, x), Y(queue, n);
    Y = X + 2 * (A * X);
    uint64_t l0 = launches();
    Y = X + 2 * (A * X);
    BOOST_CHECK_EQUAL(launches() - l0, 1u);
    check_sample(Y, [&](size_t idx, double a) { BOOST_CHECK_CLOSE(a, x[idx] + 2 * row_sum(row, col, val, x.data(), idx), 1e-8); });
    // two distinct sliced-ELL matrices: the second product goes through its temporary
    std::vector<int> row2, col2; std::vector<double> val2;
    random_matrix(n, n, 16, row2, col2, val2);
    vex::sparse::matrix<double> B(queue, n, n, row2, col2, val2);
    Y = A * X - B * X;
    check_sample(Y, [&](size_t idx, double a) {
        BOOST_CHECK_CLOSE(a, row_sum(row, col, val, x.data(), idx) - row_sum(row2, col2, val2, x.data(), idx), 1e-6);
    });
}

BOOST_AUTO_TEST_CASE(multivector_product_reads_the_strip_once)
{
    const size_t n = 4096, m = 3;
    typedef std::array<double, m> elem_t;
    std::vector<vex::command_queue> queue(1, ctx.queue(0));
    std::vector<size_t> row, col; std::vector<double> val;
    random_matrix(n, n, 16, row, col, val);
    std::vector<double> x = random_vector<double>(n * m);
    vex::SpMat<double> A(queue, n, n, row.data(), col.data(), val.data());
    BOOST_REQUIRE(A.info().loc.fmt == VEXB_FMT_SELL);
    vex::multivector<double, m> X(queue, x), Y(queue, n), Z(queue, n);
    const uint64_t l0 = launches();
    Y = A * X;
    BOOST_CHECK_EQUAL(launches() - l0, 1u);
    check_sample(Y, [&](size_t idx, elem_t a) {
        for (size_t k = 0; k < m; ++k) BOOST_CHECK_CLOSE(a[k], row_sum(row, col, val, x.data() + k * n, idx), 1e-8);
    });
    for (size_t i = 0; i < m; ++i) Z(i) = A * X(i);
    std::vector<double> y(n * m), z(n * m);
    vex::copy(Y, y); vex::copy(Z, z);
    size_t diff = 0;
    for (size_t k = 0; k < n * m; ++k) diff += y[k] != z[k];
    BOOST_CHECK_EQUAL(diff, 0u);
}
