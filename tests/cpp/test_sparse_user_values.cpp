// User value types of vex::sparse matrices: the two uses of spmv_ops_impl in the reference -- tests/sparse_matrices.cpp
// custom_values (2 x 2 blocks) and examples/complex_spmv.cpp (complex values) -- with value types of the user's own
// (structs, not std::array or std::complex), through csr, ell and matrix.  Each is checked against a host loop at 1e-8 %
// and bit for bit against the library's built-in product of the same matrix (std::array blocks, std::complex values):
// the snippets below spell the built-in kernels' arithmetic, and both are compiled without FMA contraction.
#include "testing.hpp"
#include <array>
#include <complex>
#include <cstring>
#include <vexcl/sparse/matrix.hpp>

template <class T> struct ublk { T a00, a01, a10, a11; };     // a 2 x 2 block, row-major; device T4
template <class T> struct upair { T p, q; };                  // its vector element; device T2
template <class T> struct ucplx { T re, im; };                // a complex number; device T2

namespace vex {
template <class T> struct is_cl_native<ublk<T>> : std::true_type {};
template <class T> struct is_cl_native<upair<T>> : std::true_type {};
template <class T> struct is_cl_native<ucplx<T>> : std::true_type {};
template <class T> struct type_name_impl<ublk<T>> { static std::string get() { return type_name<T>() + "4"; } };
template <class T> struct type_name_impl<upair<T>> { static std::string get() { return type_name<T>() + "2"; } };
template <class T> struct type_name_impl<ucplx<T>> { static std::string get() { return type_name<T>() + "2"; } };

namespace sparse {
template <class T> struct rhs_of<ublk<T>> { typedef upair<T> type; };

// sum_r = sum_r + (a_r0 x_0 + a_r1 x_1): the loop of custom_values
template <class T> struct spmv_ops_impl<ublk<T>, upair<T>> {
    static void decl_accum_var(backend::source_generator &src, const std::string &name) {
        src.new_line() << type_name<T>() << "2 " << name << " = {0, 0};";
    }
    static void append(backend::source_generator &src, const std::string &sum, const std::string &val) {
        src.new_line() << sum << ".x = " << sum << ".x + " << val << ".x;";
        src.new_line() << sum << ".y = " << sum << ".y + " << val << ".y;";
    }
    static void append_product(backend::source_generator &src, const std::string &sum, const std::string &mat_val,
                               const std::string &vec_val) {
        src.open("{");
        src.new_line() << type_name<T>() << " row = " << mat_val << ".x * " << vec_val << ".x + " << mat_val << ".y * " << vec_val << ".y;";
        src.new_line() << sum << ".x = " << sum << ".x + row;";
        src.new_line() << "row = " << mat_val << ".z * " << vec_val << ".x + " << mat_val << ".w * " << vec_val << ".y;";
        src.new_line() << sum << ".y = " << sum << ".y + row;";
        src.close("}");
    }
};

// (a + bi)(xr + i xi) added to the sum: the spmv_ops_impl of complex_spmv
template <class T> struct spmv_ops_impl<ucplx<T>, ucplx<T>> {
    static void decl_accum_var(backend::source_generator &src, const std::string &name) {
        src.new_line() << type_name<T>() << "2 " << name << " = {0, 0};";
    }
    static void append(backend::source_generator &src, const std::string &sum, const std::string &val) {
        src.new_line() << sum << ".x = " << sum << ".x + " << val << ".x;";
        src.new_line() << sum << ".y = " << sum << ".y + " << val << ".y;";
    }
    static void append_product(backend::source_generator &src, const std::string &sum, const std::string &mat_val,
                               const std::string &vec_val) {
        src.new_line() << sum << ".x = " << sum << ".x + (" << mat_val << ".x * " << vec_val << ".x - " << mat_val << ".y * " << vec_val << ".y);";
        src.new_line() << sum << ".y = " << sum << ".y + (" << mat_val << ".x * " << vec_val << ".y + " << mat_val << ".y * " << vec_val << ".x);";
    }
};
} // namespace sparse
} // namespace vex

template <class T> constexpr double close_pct() { return std::is_same<T, double>::value ? 1e-8 : 1e-3; }

template <class T> using bval = std::array<std::array<T, 2>, 2>;
template <class T> using bvec = std::array<T, 2>;

template <class T> static ublk<T> to_user(const bval<T> &a) { return ublk<T>{a[0][0], a[0][1], a[1][0], a[1][1]}; }
template <class T> static upair<T> to_user(const bvec<T> &v) { return upair<T>{v[0], v[1]}; }
template <class T> static ucplx<T> to_user(const std::complex<T> &z) { return ucplx<T>{z.real(), z.imag()}; }
template <class U, class B> static std::vector<U> to_user(const std::vector<B> &b) {
    std::vector<U> u; for (const B &e : b) u.push_back(to_user(e)); return u;
}

template <class A, class B> static bool same_bytes(const vex::vector<A> &a, const vex::vector<B> &b) {
    static_assert(sizeof(A) == sizeof(B), "element sizes");
    std::vector<A> ha(a.size()); std::vector<B> hb(b.size());
    vex::copy(a, ha); vex::copy(b, hb);
    return ha.size() == hb.size() && std::memcmp(ha.data(), hb.data(), ha.size() * sizeof(A)) == 0;
}

// sum over the blocks of row i, as the reference's custom_values loop
template <class T>
static bvec<T> block_row(const std::vector<int> &ptr, const std::vector<int> &col, const std::vector<bval<T>> &val,
                         const std::vector<bvec<T>> &x, size_t i) {
    bvec<T> s = {0, 0};
    for (int j = ptr[i]; j < ptr[i + 1]; j++) {
        s[0] += val[j][0][0] * x[col[j]][0] + val[j][0][1] * x[col[j]][1];
        s[1] += val[j][1][0] * x[col[j]][0] + val[j][1][1] * x[col[j]][1];
    }
    return s;
}

// the reference's custom_values case with a user block type, then `Y += A * X`; bits against the built-in block product
template <class M, class T>
static void custom_values_case(size_t n, bool tridiagonal)
{
    std::vector<vex::command_queue> q(1, ctx.queue(0));
    std::vector<int> ptr, col;
    std::vector<bval<T>> val;
    auto mconst = [](T c) { bval<T> a; for (auto &r : a) r.fill(c); return a; };
    size_t m = n;
    if (tridiagonal) {
        ptr.push_back(0);
        for (size_t i = 0; i < n; ++i) {
            if (i > 0) { col.push_back((int)i - 1); val.push_back(mconst(-1)); }
            col.push_back((int)i); val.push_back(mconst(2));
            if (i + 1 < n) { col.push_back((int)i + 1); val.push_back(mconst(-1)); }
            ptr.push_back(static_cast<int>(col.size()));
        }
    } else {
        m = 777;
        std::vector<T> scalars;
        random_matrix(n, m, 16, ptr, col, scalars);
        val.resize(col.size());
        for (auto &a : val) for (auto &r : a) for (auto &v : r) v = generator<T>::get() - T(0.5);
    }
    std::vector<bvec<T>> x(m), z(n);
    for (auto &v : x) v = tridiagonal ? bvec<T>{1, 1} : bvec<T>{generator<T>::get(), generator<T>::get()};
    for (auto &v : z) v = bvec<T>{generator<T>::get(), generator<T>::get()};

    M A(q, n, m, ptr, col, to_user<ublk<T>>(val));
    BOOST_CHECK_EQUAL(A.rows(), n);
    BOOST_CHECK_EQUAL(A.nonzeros(), val.size());
    vex::vector<upair<T>> X(q, to_user<upair<T>>(x)), Y(q, n), Z(q, to_user<upair<T>>(z));
    Y = A * X;
    Z += A * X;

    vex::sparse::matrix<bval<T>> B(q, n, m, ptr, col, val);
    vex::vector<bvec<T>> Xb(q, x), Yb(q, n), Zb(q, z);
    Yb = B * Xb;
    Zb += B * Xb;
    BOOST_CHECK(same_bytes(Y, Yb));
    BOOST_CHECK(same_bytes(Z, Zb));

    check_sample(Y, [&](size_t i, upair<T> y) {
        const bvec<T> s = block_row(ptr, col, val, x, i);
        BOOST_CHECK_CLOSE(y.p, s[0], close_pct<T>());
        BOOST_CHECK_CLOSE(y.q, s[1], close_pct<T>());
        if (tridiagonal) {
            const T want = (i == 0 || i == n - 1) ? T(2) : T(0);
            BOOST_CHECK_EQUAL(y.p, want);
            BOOST_CHECK_EQUAL(y.q, want);
        }
    });
    check_sample(Z, [&](size_t i, upair<T> y) {
        const bvec<T> s = block_row(ptr, col, val, x, i);
        BOOST_CHECK_CLOSE(y.p, z[i][0] + s[0], close_pct<T>());
        BOOST_CHECK_CLOSE(y.q, z[i][1] + s[1], close_pct<T>());
    });
}

// the body of the reference's complex_spmv example with a user complex type; bits against the built-in complex product
template <class M>
static void complex_example_case()
{
    std::vector<vex::command_queue> q(1, ctx.queue(0));
    std::vector<int> ptr = {0, 1, 2, 3, 4};
    std::vector<int> col = {0, 1, 2, 3};
    std::vector<std::complex<double>> val = {{1.0, 1.0}, {2.0, 2.0}, {3.0, 3.0}, {4.0, 4.0}};
    std::vector<std::complex<double>> x = {{1.0, 1.0}, {1.0, 1.0}, {1.0, 1.0}, {1.0, 1.0}};

    M A(q, 4, 4, ptr, col, to_user<ucplx<double>>(val));
    vex::vector<ucplx<double>> X(q, to_user<ucplx<double>>(x));
    vex::vector<ucplx<double>> Y(q, 4);
    Y = A * X;
    for (int k = 0; k < 4; ++k) {                          // (k+1)(1+i) * (1+i) = 2(k+1) i, exactly
        ucplx<double> y = Y[k];
        BOOST_CHECK_EQUAL(y.re, 0.0);
        BOOST_CHECK_EQUAL(y.im, 2.0 * (k + 1));
    }
    vex::sparse::matrix<std::complex<double>> Zm(q, 4, 4, ptr, col, val);
    vex::vector<std::complex<double>> Xz(q, x), Yz(q, 4);
    Yz = Zm * Xz;
    BOOST_CHECK(same_bytes(Y, Yz));
}

template <class M, class T>
static void complex_random_case()
{
    typedef std::complex<T> Zt;
    const size_t n = 1024, m = 777;
    std::vector<vex::command_queue> q(1, ctx.queue(0));
    std::vector<int> ptr, col; std::vector<T> scalars;
    random_matrix(n, m, 16, ptr, col, scalars);
    std::vector<Zt> val(col.size()), x(m), z(n);
    for (auto &a : val) a = Zt(generator<T>::get() - T(0.5), generator<T>::get() - T(0.5));
    for (auto &v : x) v = Zt(generator<T>::get(), generator<T>::get());
    for (auto &v : z) v = Zt(generator<T>::get(), generator<T>::get());

    M A(q, n, m, ptr, col, to_user<ucplx<T>>(val));
    vex::vector<ucplx<T>> X(q, to_user<ucplx<T>>(x)), Y(q, n), Z(q, to_user<ucplx<T>>(z));
    Y = A * X;
    Z += A * X;
    vex::sparse::matrix<Zt> C(q, n, m, ptr, col, val);
    vex::vector<Zt> Xc(q, x), Yc(q, n), Zc(q, z);
    Yc = C * Xc;
    Zc += C * Xc;
    BOOST_CHECK(same_bytes(Y, Yc));
    BOOST_CHECK(same_bytes(Z, Zc));
    check_sample(Y, [&](size_t i, ucplx<T> y) {
        T re = 0, im = 0;
        for (int j = ptr[i]; j < ptr[i + 1]; j++) {
            re += val[j].real() * x[col[j]].real() - val[j].imag() * x[col[j]].imag();
            im += val[j].real() * x[col[j]].imag() + val[j].imag() * x[col[j]].real();
        }
        BOOST_CHECK_CLOSE(y.re, re, close_pct<T>());
        BOOST_CHECK_CLOSE(y.im, im, close_pct<T>());
    });
}

BOOST_AUTO_TEST_CASE(custom_values)
{
    custom_values_case<vex::sparse::matrix<ublk<double>>, double>(1024, true);
    custom_values_case<vex::sparse::csr<ublk<double>>, double>(1024, true);
    custom_values_case<vex::sparse::ell<ublk<double>>, double>(1024, true);
}

BOOST_AUTO_TEST_CASE(user_blocks_random)
{
    custom_values_case<vex::sparse::matrix<ublk<double>>, double>(1024, false);
    custom_values_case<vex::sparse::csr<ublk<float>>, float>(1024, false);
    custom_values_case<vex::sparse::ell<ublk<float>>, float>(3000, false);
}

BOOST_AUTO_TEST_CASE(complex_spmv_example)
{
    complex_example_case<vex::sparse::matrix<ucplx<double>>>();
    complex_example_case<vex::sparse::csr<ucplx<double>>>();
    complex_example_case<vex::sparse::ell<ucplx<double>>>();
}

BOOST_AUTO_TEST_CASE(user_complex_random)
{
    complex_random_case<vex::sparse::matrix<ucplx<double>>, double>();
    complex_random_case<vex::sparse::csr<ucplx<float>>, float>();
}

BOOST_AUTO_TEST_CASE(user_matrix_needs_one_device)
{
    std::vector<int> ptr = {0, 1}, col = {0};
    std::vector<ucplx<double>> val(1, ucplx<double>{1, 1});
    std::vector<vex::command_queue> q2(2, ctx.queue(0));
    BOOST_CHECK_THROW(vex::sparse::matrix<ucplx<double>> A(q2, 1, 1, ptr, col, val), std::exception);
}
