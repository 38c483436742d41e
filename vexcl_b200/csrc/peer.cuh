// One-hop all-reduce over NVLink peer memory, callable from inside a kernel: the protocol and its device side
// (PeerArgs, peer_exchange, peer_poison) live in fold.cuh, next to the reduction finish that calls them, because the
// NVRTC-generated reductions embed that text too.  This header adds the host side: the group handle vexb_peer.
#pragma once
#include "common.cuh"
#include "fold.cuh"

namespace vexb {

// Process-wide sticky fault word in mapped pinned host memory (peer.cu): 0 = no fault.
unsigned long long *peer_fault_word();

} // namespace vexb

struct vexb_peer {
    int dev = 0, rank = 0, nranks = 1;
    unsigned long long *mailbox = nullptr;                  // mine
    unsigned long long *peers[VEXB_MAX_PEERS] = {nullptr};  // everybody's, as mapped here
    bool ipc_opened[VEXB_MAX_PEERS] = {false};
    unsigned long long *fault_host = nullptr;
    vexb::PeerArgs args() const {
        vexb::PeerArgs a; a.rank = rank; a.nranks = nranks; a.fault_host = fault_host;
        for (int p = 0; p < VEXB_MAX_PEERS; ++p) a.mbox[p] = p < nranks ? peers[p] : nullptr;
        return a;
    }
};
