// The slice of a multi-device vex::SpMat owned by one device (internal layout shared by dspmat.cu and distapply.cu).
#pragma once
#include "spmat.hpp"
#include <vector>

namespace vexb { struct HaloLink; }
struct vexb_peer;

struct vexb_dspmat {
    int dev = 0, part = 0, nparts = 1, val_dtype = VEXB_F64;
    bool values_f32 = false;        // created with VEXB_FMT_VALUES_F32: no peer-memory halo, no fused product + dot
    size_t nrows = 0, ncols_local = 0, n_ghost = 0, n_send = 0;
    vexb_spmat *loc = nullptr;      // rows without ghost entries (all rows when there are no ghosts)
    vexb_spmat *bnd = nullptr;      // local entries of the rows that also have ghost entries (row-compressed)
    vexb_spmat *rem = nullptr;      // ghost entries of those rows (row-compressed)
    int *send_cols = nullptr;       // device: local x indices to pack, grouped by destination
    void *send_buf = nullptr;       // device: n_send values
    void *ghost_buf = nullptr;      // device: n_ghost values ("rx" of spmat.hpp:273)
    std::vector<size_t> send_counts, recv_counts;
    cudaStream_t side = nullptr;    // secondary queue (spmat.hpp:81-82)
    cudaEvent_t ev_pack = nullptr, ev_halo = nullptr, ev_x = nullptr;
    // host copies of the split, kept for parity checks
    std::vector<int64_t> loc_ptr, loc_col, rem_ptr, rem_col;
    std::vector<char> loc_val, rem_val;
    size_t loc_nnz = 0, rem_nnz = 0; bool split_kept = false;
    vexb::HaloLink *halo = nullptr; // peer-memory halo (distapply.cu): set by vexb_dspmat_halo_connect*, NULL = NCCL / copies
    std::vector<size_t> ghost_counts;        // n_ghost of every part (from the plan)
    std::vector<size_t> land_off;            // land_off[p]: where my values start in part p's ghost buffer
};


namespace vexb {
// distapply.cu: the peer-memory halo and the fused apply kernel
void halo_link_destroy(HaloLink *h);
int halo_prepare(vexb_dspmat *A);
int dist_apply(const vexb_dspmat *A, cudaStream_t st, const void *x, void *y, double alpha, int append, const void *dot_with,
               void *dot_result, const vexb_peer *peer);
int halo_set_boundary(vexb_dspmat *A, const std::vector<int> &rows, int width, const std::vector<int> &col, const void *val);
}
