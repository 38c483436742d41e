// Block values of vex::sparse matrices: the reference's tests/sparse_matrices.cpp custom_values case (:239-282) against
// include/vexcl/sparse, then the same case for 3x3 and 4x4 blocks and for float, a random block matrix, and
// `Y += A * X` / `Y -= A * X`, each for csr, ell and matrix.
#include "testing.hpp"
#include <array>
#include <vexcl/sparse/matrix.hpp>
#include <vexcl/sparse/distributed.hpp>

typedef std::array<std::array<double, 2>, 2> matrix_value;
typedef std::array<double, 2> vector_value;

// The reference's own rhs_of specialisation still compiles (and agrees with the library's).  Its is_cl_native,
// type_name_impl and spmv_ops_impl specialisations teach its source generator the types; this front end has no
// generator and knows B x B blocks from their type, so they are left out.
namespace vex { namespace sparse {
template <> struct rhs_of<matrix_value> { typedef vector_value type; };
} }

template <class T, size_t B> using mval = std::array<std::array<T, B>, B>;
template <class T, size_t B> using vval = std::array<T, B>;

template <class T, size_t B> mval<T, B> mconst(T c) { mval<T, B> a; for (auto &r : a) r.fill(c); return a; }
template <class T, size_t B> vval<T, B> vconst(T c) { vval<T, B> v; v.fill(c); return v; }

template <class T> constexpr double close_pct() { return std::is_same<T, double>::value ? 1e-8 : 1e-4; }

// sum[r] over the blocks of row i, in the order of the reference loop (sparse_matrices.cpp:274-277)
template <class T, size_t B>
static vval<T, B> row_product(const std::vector<int> &ptr, const std::vector<int> &col, const std::vector<mval<T, B>> &val,
                              const std::vector<vval<T, B>> &x, size_t i) {
    vval<T, B> sum = vconst<T, B>(0);
    for (int j = ptr[i]; j < ptr[i + 1]; j++)
        for (size_t r = 0; r < B; ++r) {
            T t = val[j][r][0] * x[col[j]][0];
            for (size_t q = 1; q < B; ++q) t = t + val[j][r][q] * x[col[j]][q];
            sum[r] += t;
        }
    return sum;
}

template <class M, class T, size_t B>
static void custom_values_case()
{
    const int n = 1024;
    std::vector<vex::command_queue> q(1, ctx.queue(0));

    std::vector<int> ptr, col;
    std::vector<mval<T, B>> val;

    ptr.push_back(0);
    for (int i = 0; i < n; ++i) {
        if (i > 0) { col.push_back(i - 1); val.push_back(mconst<T, B>(-1)); }
        col.push_back(i); val.push_back(mconst<T, B>(2));
        if (i + 1 < n) { col.push_back(i + 1); val.push_back(mconst<T, B>(-1)); }
        ptr.push_back(static_cast<int>(col.size()));
    }

    M A(q, n, n, ptr, col, val);
    BOOST_CHECK_EQUAL(A.rows(), static_cast<size_t>(n));
    BOOST_CHECK_EQUAL(A.nonzeros(), val.size());

    std::vector<vval<T, B>> x(n, vconst<T, B>(1));
    vex::vector<vval<T, B>> X(q, x);
    vex::vector<vval<T, B>> Y(q, n);

    Y = A * X;

    for (int i = 0; i < n; ++i) {                          // all rows, as the reference does
        vval<T, B> y = Y[i];
        vval<T, B> sum = row_product(ptr, col, val, x, i);
        for (size_t r = 0; r < B; ++r) BOOST_CHECK_CLOSE(y[r], sum[r], 1e-8);
        for (size_t r = 0; r < B; ++r) BOOST_CHECK_EQUAL(y[r], (i == 0 || i == n - 1) ? T(B) : T(0));
    }
}

template <class M, class T, size_t B>
static void random_case()
{
    const size_t n = 1024, m = 777;
    std::vector<vex::command_queue> q(1, ctx.queue(0));
    std::vector<int> ptr, col; std::vector<T> scalars;
    random_matrix(n, m, 16, ptr, col, scalars);
    std::vector<mval<T, B>> val(col.size());
    for (auto &a : val) for (auto &r : a) for (auto &v : r) v = generator<T>::get() - T(0.5);
    std::vector<vval<T, B>> x(m), z(n);
    for (auto &v : x) for (auto &e : v) e = generator<T>::get();
    for (auto &v : z) for (auto &e : v) e = generator<T>::get();

    M A(q, n, m, ptr, col, val);
    BOOST_CHECK_EQUAL(A.cols(), m);
    vex::vector<vval<T, B>> X(q, x), Y(q, n), Z(q, z);

    Y = A * X;
    check_sample(Y, [&](size_t i, vval<T, B> y) {
        vval<T, B> sum = row_product(ptr, col, val, x, i);
        for (size_t r = 0; r < B; ++r) BOOST_CHECK_CLOSE(y[r], sum[r], close_pct<T>());
    });

    Z += A * X;                                           // z + s
    check_sample(Z, [&](size_t i, vval<T, B> y) {
        vval<T, B> sum = row_product(ptr, col, val, x, i);
        for (size_t r = 0; r < B; ++r) BOOST_CHECK_CLOSE(y[r], z[i][r] + sum[r], close_pct<T>());
    });
    Z -= A * X;
    Z -= A * X;                                           // (z + s) - s - s
    check_sample(Z, [&](size_t i, vval<T, B> y) {
        vval<T, B> sum = row_product(ptr, col, val, x, i);
        for (size_t r = 0; r < B; ++r) {
            const T want = (z[i][r] + sum[r]) - sum[r] - sum[r];
            BOOST_CHECK_SMALL(y[r] - want, 1e-5 * (std::fabs(z[i][r]) + 3 * std::fabs(sum[r]) + 1));
        }
    });

    // the vectors' bytes are B values per element, in order (vex::copy and element reads agree)
    std::vector<vval<T, B>> back(n);
    vex::copy(Z, back);
    for (size_t i = 0; i < n; i += 101) { vval<T, B> e = Z[i]; BOOST_CHECK(e == back[i]); }
}

template <class T, size_t B>
static void all_formats() {
    custom_values_case<vex::sparse::csr<mval<T, B>>, T, B>();
    custom_values_case<vex::sparse::ell<mval<T, B>>, T, B>();
    custom_values_case<vex::sparse::matrix<mval<T, B>>, T, B>();
    random_case<vex::sparse::csr<mval<T, B>>, T, B>();
    random_case<vex::sparse::ell<mval<T, B>>, T, B>();
    random_case<vex::sparse::matrix<mval<T, B>>, T, B>();
}

BOOST_AUTO_TEST_CASE(custom_values)
{
    // the reference's case as it is written there: 2x2 double blocks through vex::sparse::matrix
    custom_values_case<vex::sparse::matrix<matrix_value>, double, 2>();
    static_assert(std::is_same<vex::sparse::rhs_of<matrix_value>::type, vector_value>::value, "rhs_of");
    static_assert(std::is_same<vex::sparse::rhs_of<mval<float, 3>>::type, vval<float, 3>>::value, "rhs_of");
    static_assert(std::is_same<vex::sparse::rhs_of<double>::type, double>::value, "rhs_of");
}

BOOST_AUTO_TEST_CASE(blocks_2_double) { all_formats<double, 2>(); }
BOOST_AUTO_TEST_CASE(blocks_3_double) { all_formats<double, 3>(); }
BOOST_AUTO_TEST_CASE(blocks_4_double) { all_formats<double, 4>(); }
BOOST_AUTO_TEST_CASE(blocks_2_float)  { all_formats<float, 2>(); }
BOOST_AUTO_TEST_CASE(blocks_3_float)  { all_formats<float, 3>(); }
BOOST_AUTO_TEST_CASE(blocks_4_float)  { all_formats<float, 4>(); }

BOOST_AUTO_TEST_CASE(block_matrix_needs_one_device)
{
    // like the scalar classes: a context of two queues is refused at construction
    std::vector<int> ptr = {0, 1}, col = {0};
    std::vector<matrix_value> val(1, mconst<double, 2>(1));
    std::vector<vex::command_queue> q2(2, ctx.queue(0));
    BOOST_CHECK_THROW(vex::sparse::matrix<matrix_value> A(q2, 1, 1, ptr, col, val), std::exception);
}
