// Device-resident sparse strip (internal layout shared by spmv.cu and dspmat.cu).
#pragma once
#include "hostlogic.hpp"
#include <vector>

namespace vexb {
// 16-bit ELL columns are stored as distances from (row + shift of the slot): one shift per ELL slot (a 7-point stencil
// has its neighbours n*n, n, 1 away -- no single shift brings them all within 16 bits, one shift per slot does).  Slots
// past the last entry share it.
constexpr int kEllShiftSlots = 16;
// x_max: largest column the strip stores, set on row-class strips only (EllClass below).
struct EllShifts { int s[kEllShiftSlots]; int x_max; };
// Widths for which EVERY kernel that walks an ELL strip has an unrolled instantiation (hell_kernel, hell_multi_kernel,
// dist_apply_kernel: keep their switches in step with this).  Only those strips get one shift per slot: the kernels'
// run-time loop over the slots reads shift.s[0] for all of them (indexing the by-value table at run time spills it).
constexpr bool ell_width_is_unrolled_everywhere(size_t w) { return w == 3 || w == 5 || w == 7 || w == 9; }
// Column type of the third ELL encoding (spmv.ell_diag): no column array.  Every entry of slot k sits at (row + shift of
// slot k), so a row stores only which of its slots hold an entry: bit k of its mask.  The kernels take a pointer to the
// per-row masks where the other encodings pass their column array.
constexpr size_t kEllDiagMaxWidth = 8;
struct EllDiag { unsigned char mask; };
// Column type of the fourth ELL encoding (spmv.ell_classes): a slot-mask strip whose rows take at most kEllMaxClasses
// distinct (slot mask, W slot values) tuples -- any constant-coefficient stencil -- stores one class byte per row and no
// per-slot values.  The kernels take the class bytes where they take masks and the class table where they take the
// values.  Class table, in device memory: kEllClassHeader bytes of slot masks (one per class), then W values per class.
constexpr size_t kEllMaxClasses = 256;
constexpr size_t kEllClassHeader = 256;
struct EllClass { unsigned char id; };
}

struct vexb_spmat {
    int dev = 0;
    int fmt = VEXB_FMT_CSR;
    int val_dtype = VEXB_F64;
    bool val_f32 = false;          // VEXB_FMT_VALUES_F32: val, sell_val, ell_val and tail_val hold float (x, y, sums: double)
    size_t nrows = 0, ncols = 0, nnz = 0;
    // CSR stream
    void *val = nullptr; int *col = nullptr; int *rowptr = nullptr; int2 *tile = nullptr;
    size_t n_tiles = 0, tile_nnz = 0, tile_rows = 0;
    int2 *tile_x = nullptr; size_t xwin = 0, n_windowed_tiles = 0;   // per CTA tile: {first column, length} of its x window (csr_window_kernel)
    int2 *wtile = nullptr; size_t n_wtiles = 0;   // warp tiles (<= 256 nnz, <= 256 rows) for csr_warp_kernel
    int csr_variant = 0;                          // kernel picked for this strip when spmv.kernel is not set (see build())
    size_t max_row_nnz = 0;
    // HELL
    size_t ell_width = 0, ell_pitch = 0, tail_nnz = 0;
    int *ell_col = nullptr; void *ell_val = nullptr;
    short *ell_col16 = nullptr; vexb::EllShifts ell_shifts = {};   // optional: columns as 16-bit offsets from (row + shift of the slot); see spmv.col16
    vexb::EllDiag *ell_mask = nullptr;   // optional: one slot mask per stored row, column of slot k = row + ell_shifts.s[k]; see spmv.ell_diag
    // optional: one class id per stored row and the class table in place of ell_mask and ell_val; see spmv.ell_classes
    vexb::EllClass *ell_class = nullptr; void *ell_ctab = nullptr; size_t ell_nclass = 0;
    // exactly one of ell_col / ell_col16 / ell_mask / ell_class is set on a HELL strip of width > 0
    const void *ell_col_any() const {
        return ell_class ? (const void *)ell_class : ell_mask ? (const void *)ell_mask : ell_col16 ? (const void *)ell_col16 : (const void *)ell_col;
    }
    const void *ell_val_any() const { return ell_class ? ell_ctab : ell_val; }
    int *tail_ptr = nullptr; int *tail_col = nullptr; void *tail_val = nullptr;
    // SELL-32-sigma: slice s holds stored rows perm[32 s .. 32 s + 31] (-1: none) in sell_col / sell_val at
    // [slice_ptr[s], slice_ptr[s+1]), slot k of lane l at slice_ptr[s] + 32 k + l
    int *sell_ptr = nullptr; int *sell_perm = nullptr; int *sell_col = nullptr; void *sell_val = nullptr;
    short *sell_col16 = nullptr; int sell_shift = 0;   // optional 16-bit columns: distance from (row + sell_shift), -32768 = padding
    size_t n_slices = 0, sell_slots = 0;
    vexb_ccsr *patterns = nullptr; // VEXB_FMT_PATTERNS: the strip as unique row patterns + one pattern id per row (csrc/ccsr.cu)
    size_t n_patterns = 0;
    int *row_ids = nullptr;        // optional: compressed rows, y index of stored row r (remote strips)
    size_t y_offset = 0;           // y index of stored row 0 when the strip covers a contiguous row range
    size_t nrows_stored = 0;       // rows held in the arrays (== nrows unless row_ids)
    size_t device_bytes = 0;
    void *d_desc = nullptr;        // device copy of vexb::SpmvDesc (what a generated kernel needs to walk the rows); see jit.cu
};

namespace vexb {
// Everything a kernel generated for a VEXB_TERM_SPMV terminal reads about the strip (uniform loads through one pointer).
struct SpmvDesc {
    const void *ell_col;   // vexb_spmat::ell_col_any(): 32-bit columns, 16-bit offsets, slot masks or class ids
    const void *ell_val;   // vexb_spmat::ell_val_any(): values, or the class table
    const int *tail_ptr; const int *tail_col; const void *tail_val;
    const int *rowptr; const int *col; const void *val;
    unsigned long long pitch; int width; int shifts[kEllShiftSlots]; int x_max;
    // sliced ELL: what sell_kernel takes (sell_col: 16-bit offsets when the strip has them, else 32-bit columns)
    const int *slice_ptr; const int *perm; const void *sell_col; const void *sell_val; int sell_shift; unsigned long long n_slices;
};
}

namespace vexb {
// Build a strip from 32-bit host CSR.  row_ids (optional) maps stored row r to its y index;
// nrows is then the length of y and rowptr.size()-1 the number of stored rows.
// fmt may carry VEXB_FMT_VALUES_F32; val must then already be rounded to float (round_values_f32).
int spmat_from_csr(int dev, size_t nrows, size_t ncols, std::vector<int> &rowptr, std::vector<int> &col,
                   const void *val, int val_dtype, int fmt, const std::vector<int> *row_ids, vexb_spmat **out);
// Checks the flag bits of `fmt` against val_dtype and, with VEXB_FMT_VALUES_F32, fills `rounded` with double(float(v)) of
// the n values (exact both ways, as numpy's astype(float32)); VEXB_ERR_INVALID when a finite value rounds to +-inf.
// Host only: the create functions call it before they touch a device.
int check_fmt_flags(int fmt, int val_dtype, const void *val, size_t n, std::vector<double> &rounded);
}
