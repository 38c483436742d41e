#ifndef VEXCL_SPARSE_SPMV_OPS_HPP
#define VEXCL_SPARSE_SPMV_OPS_HPP
/*
 * vex::sparse::spmv_ops_impl<mat_type, vec_type> (vexcl/sparse/spmv_ops.hpp): the device code of a sparse product whose
 * values are a user type.  A specialisation writes three snippets into a backend::source_generator:
 *   decl_accum_var(src, sum)                    declares the accumulator `sum`, zeroed;
 *   append_product(src, sum, mat_val, vec_val)  adds the product of one stored value and x at its column to `sum`;
 *   append(src, sum, val)                       adds `val` to `sum` (y += A * x).
 * sparse/matrix.hpp builds them once per matrix with the names sum, v, xv and t, and the library compiles them into a
 * sliced-ELL kernel for sm_90a (vexb_usr_spmv) with --fmad=false: every product and sum in a snippet is rounded on its
 * own, in the order written.  The types named in the snippets are those NVRTC knows (double2, double4, float2, ...).
 *
 * Only user value types (vex::is_user_value) go through these snippets.  Scalars, B x B std::array blocks and
 * std::complex values have kernels of their own; a specialisation for them compiles but is not used.
 */
#include <string>
#include "../backend.hpp"
#include "../types.hpp"

namespace vex {
namespace sparse {

template <class mat_type, class vec_type, class enable = void>
struct spmv_ops_impl {
    static_assert(sizeof(mat_type) == 0, "a sparse matrix of a user value type needs a specialisation of "
                  "vex::sparse::spmv_ops_impl<value type, rhs_of<value type>::type> with static decl_accum_var, "
                  "append_product and append");
    static void decl_accum_var(backend::source_generator&, const std::string&) {}
    static void append(backend::source_generator&, const std::string&, const std::string&) {}
    static void append_product(backend::source_generator&, const std::string&, const std::string&, const std::string&) {}
};

} // namespace sparse
} // namespace vex
#endif
