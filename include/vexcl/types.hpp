#ifndef VEXCL_TYPES_HPP
#define VEXCL_TYPES_HPP
// Element types understood by the back end and their names (subset of vexcl/types.hpp:202-260:
// scalars only -- OpenCL vector types are outside the hot path).
#include <array>
#include <complex>
#include <cstdint>
#include <string>
#include <type_traits>
#include "../vexb200.h"

typedef unsigned int  uint;
typedef double        cl_double;
typedef float         cl_float;
typedef int           cl_int;
typedef unsigned int  cl_uint;
typedef long long     cl_long;
typedef unsigned long long cl_ulong;

namespace vex {

/// N-component result of combined reductions (stands in for cl_double2 / cl_double4 / ...; fields as in CL: s[0], s[1], ...).
template <class T, unsigned N> struct vecn { T s[N]; };
template <class T> using vec2 = vecn<T, 2>;
/// Smallest CL vector width that holds n components (vexcl/types.hpp cl_fit_vec_size): 1, 2, 4, 8 or 16.
template <unsigned n> struct cl_fit_vec_size { static const unsigned value = n <= 1 ? 1 : n <= 2 ? 2 : n <= 4 ? 4 : n <= 8 ? 8 : 16; };

/// Declares a type usable as a vector element and a sparse matrix value (vexcl/types.hpp).  Arithmetic types are; a
/// user type V that is specialised true here (and has a vex::sparse::spmv_ops_impl) is a user value type, below.
template <class T> struct is_cl_native : std::is_arithmetic<T> {};

namespace detail {
template <class T> struct is_std_array : std::false_type {};
template <class T, size_t N> struct is_std_array<std::array<T, N>> : std::true_type {};
template <class T> struct is_std_complex : std::false_type {};
template <class T> struct is_std_complex<std::complex<T>> : std::true_type {};
}

/// A user value type: declared by is_cl_native, neither arithmetic nor a block (std::array) nor std::complex, which have
/// kernels of their own.  Sparse matrices of it multiply through its spmv_ops_impl (sparse/spmv_ops.hpp, sparse/matrix.hpp).
template <class T> struct is_user_value
    : std::integral_constant<bool, is_cl_native<T>::value && !std::is_arithmetic<T>::value && !detail::is_std_array<T>::value &&
                                   !detail::is_std_complex<T>::value> {};

template <class T, class Enable = void> struct dtype_of;   // no definition: unsupported element type
#define VEXB_DTYPE(T, code, nm) \
    template <> struct dtype_of<T> { static const int value = code; static const char *name() { return nm; } };
VEXB_DTYPE(double, VEXB_F64, "double")
VEXB_DTYPE(float, VEXB_F32, "float")
VEXB_DTYPE(int, VEXB_I32, "int")
VEXB_DTYPE(unsigned int, VEXB_U32, "uint")
VEXB_DTYPE(long, VEXB_I64, "long")
VEXB_DTYPE(unsigned long, VEXB_U64, "ulong")
VEXB_DTYPE(long long, VEXB_I64, "long")
VEXB_DTYPE(unsigned long long, VEXB_U64, "ulong")
#undef VEXB_DTYPE
// small integers and bool appear only as scalar terminals: promoted to int, as C does
template <> struct dtype_of<bool>  { static const int value = VEXB_I32; static const char *name() { return "bool"; } };
template <> struct dtype_of<char>  { static const int value = VEXB_I32; static const char *name() { return "char"; } };
template <> struct dtype_of<short> { static const int value = VEXB_I32; static const char *name() { return "short"; } };
template <> struct dtype_of<signed char>    { static const int value = VEXB_I32; static const char *name() { return "char"; } };
template <> struct dtype_of<unsigned char>  { static const int value = VEXB_I32; static const char *name() { return "uchar"; } };
template <> struct dtype_of<unsigned short> { static const int value = VEXB_I32; static const char *name() { return "ushort"; } };

// std::array<T, B> is the element of block vectors, vex::vector<std::array<T, B>> (and std::array<std::array<T, B>, B> the
// value of block sparse matrices, sparse/matrix.hpp).  Block products write them with one call of their own; no
// expression kernel takes them, so naming their element type is the point where any other use fails to compile.
template <class T, size_t N> struct dtype_of<std::array<T, N>> {
    static_assert(sizeof(T) == 0, "vex::vector<std::array<T, B>> holds block vectors: the only expressions on them are "
                                  "Y = A * X, Y += A * X and Y -= A * X with a block matrix vex::sparse::{csr, ell, matrix}"
                                  "<std::array<std::array<T, B>, B>>");
    static const int value = -1;
    static const char *name() { return "block"; }
};

// std::complex<T> is the element of complex vectors, vex::vector<std::complex<T>>, and the value of complex sparse matrices
// (sparse/matrix.hpp): as with blocks, only their products write them.
template <class T> struct dtype_of<std::complex<T>> {
    static_assert(sizeof(T) == 0, "vex::vector<std::complex<T>> holds complex vectors: the only expressions on them are "
                                  "Y = A * X, Y += A * X and Y -= A * X with a complex matrix vex::sparse::{csr, ell, matrix}"
                                  "<std::complex<T>>");
    static const int value = -1;
    static const char *name() { return "complex"; }
};

// User value types are the element of vex::vector<X> and the value of sparse matrices of them (sparse/matrix.hpp): as with
// blocks, only their products write them.
template <class T> struct dtype_of<T, typename std::enable_if<is_user_value<T>::value>::type> {
    static_assert(sizeof(T) == 0, "vex::vector<T> of a user value type (is_cl_native<T>) holds values no expression kernel "
                                  "knows: the only expressions on them are Y = A * X and Y += A * X with a vex::sparse::{csr, "
                                  "ell, matrix} of a user value type");
    static const int value = -1;
    static const char *name() { return "user"; }
};

/// Device name of a type (vexcl/types.hpp type_name_impl).  The built-in scalars keep the names of dtype_of; users
/// specialise it for their value types, whose names go into the generated sparse product kernel (spmv_ops.hpp).
template <class T, class Enable = void> struct type_name_impl {
    static std::string get() {
        static_assert(!is_user_value<T>::value, "a user value type needs a specialisation of vex::type_name_impl<T> whose "
                                                "get() returns its device type name");
        return dtype_of<T>::name();
    }
};

template <class T> inline std::string type_name() { return type_name_impl<typename std::decay<T>::type>::get(); }

template <class T> struct cl_scalar_of { typedef T type; };
template <class T> struct cl_vector_length { static const unsigned value = 1; };

} // namespace vex
#endif
