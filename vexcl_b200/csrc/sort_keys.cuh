// The order of vexb_sort and vexb_sort_merge, in one place: a key maps to unsigned "ordered bits" whose unsigned order
// is the sort order.  The radix passes (csrc/sort.cu) take their digits from these bits, and the host merge of sorted
// parts compares them, so the device and the host can never disagree.
//
//   unsigned keys   identity
//   signed keys     sign bit flipped
//   floating keys   -0.0 -> +0.0 and every NaN -> one positive quiet NaN (so they compare equal, above +inf), then
//                   negative values all bits flipped, the others the sign bit set
//   descending      the result XORed with all ones (desc_mask = ~0; 0 for ascending)
//
// Only the order uses these bits: the sort writes each key back with its original bits.
#pragma once
#include <cstdint>
#include "../../include/vexb200.h"

namespace vexb {

template <int DT> struct sort_bits { typedef uint32_t type; };
template <> struct sort_bits<VEXB_F64> { typedef uint64_t type; };
template <> struct sort_bits<VEXB_I64> { typedef uint64_t type; };
template <> struct sort_bits<VEXB_U64> { typedef uint64_t type; };

template <int DT>
__host__ __device__ __forceinline__ typename sort_bits<DT>::type
sort_order(typename sort_bits<DT>::type u, typename sort_bits<DT>::type desc_mask) {
    typedef typename sort_bits<DT>::type U;
    constexpr U sign = U(1) << (8 * sizeof(U) - 1);
    if constexpr (DT == VEXB_F32 || DT == VEXB_F64) {
        constexpr U exp = DT == VEXB_F32 ? U(0x7F800000u) : U(0x7FF0000000000000ull);
        constexpr U quiet = DT == VEXB_F32 ? U(0x00400000u) : U(0x0008000000000000ull);
        if ((u & ~sign) > exp) u = exp | quiet;         // any NaN
        if (u == sign) u = 0;                           // -0.0
        u = (u & sign) ? ~u : (u | sign);
    } else if constexpr (DT == VEXB_I32 || DT == VEXB_I64) {
        u ^= sign;
    }
    return u ^ desc_mask;
}

} // namespace vexb
