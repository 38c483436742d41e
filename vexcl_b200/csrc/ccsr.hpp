// Internal entry points of the CCSR code: creation shared with spmv.cu (row-pattern strips of vex::SpMat), and what the
// generated kernels of jit.cu need to take a matrix as a VEXB_TERM_CCSR terminal.
#pragma once
#include <cstddef>
#include "../../include/vexb200.h"

namespace vexb {
/// vexb_ccsr_create for a matrix whose rows index a vector of `xlen` elements (the public call has xlen = n).
int ccsr_create_ex(int dev, size_t n, size_t xlen, size_t m, const void *idx, int idx_bytes,
                   const void *row, int row_bytes, const void *col, int col_bytes,
                   const void *val, int val_dtype, vexb_ccsr **out);
/// The checks of a VEXB_TERM_CCSR terminal (term slot k) against its handle: device, value type, idx width, and a call
/// that covers the whole matrix.
int ccsr_term_check(const vexb_ccsr *A, int k, int dev, int dtype, int idx_bytes, size_t n, size_t index_offset);
/// The device descriptor {idx, row, col, val} a generated row loop reads; allocated at the first call (blocking copy).
int ccsr_term_desc(const vexb_ccsr *A, void **desc);
}
