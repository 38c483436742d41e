#ifndef VEXCL_VEXCL_HPP
#define VEXCL_VEXCL_HPP
// Umbrella header, as vexcl/vexcl.hpp in the reference: the three hot paths behind their
// original spellings, backed by libvexb200.so (link with -lvexb200).
#include <algorithm>
#include "backend.hpp"
#include "util.hpp"
#include "types.hpp"
#include "devlist.hpp"
#include "profiler.hpp"
#include "operations.hpp"
#include "vector.hpp"
#include "multivector.hpp"
#include "function.hpp"
#include "element_index.hpp"
#include "constants.hpp"
#include "tagged_terminal.hpp"
#include "temporary.hpp"
#include "vector_pointer.hpp"
#include "reductor.hpp"
#include "sort.hpp"
#include "scan.hpp"
#include "scan_by_key.hpp"
#include "reduce_by_key.hpp"
#include "spmat.hpp"
#include "spmat/ccsr.hpp"
#include "stencil.hpp"
#include "sparse/product.hpp"
#include "sparse/matrix.hpp"
#include "sparse/distributed.hpp"

namespace vex {
using backend::command_queue;
// Kernel caches and compile options have no meaning here (the library keeps its own caches and options); kept as
// no-ops so existing programs build (cache.hpp:170-183, backend/common.hpp:111-206).  So are the one-argument header
// calls; the per-queue ones below are real.
inline void purge_caches() {}
inline void purge_caches(const std::vector<backend::command_queue>&) {}
inline void push_compile_options(const std::string&) {}
inline void pop_compile_options() {}
inline void push_program_header(const std::string&) {}
inline void pop_program_header() {}

// Program headers (backend/common.hpp:120-206): text at the very top of every kernel the library compiles at run time
// for a device from user text -- expressions that call a VEX_FUNCTION, VEX_STENCIL_OPERATOR, user value types of
// vex::sparse.  A push replaces the device's header, a pop restores the previous one.  The library keeps one stack per
// device, so a queue list pushes and pops once per distinct device (two queues on one device share its header).
namespace detail {
inline std::vector<int> header_devices(const std::vector<backend::command_queue> &queue) {
    std::vector<int> devs;
    for (const auto &q : queue)
        if (std::find(devs.begin(), devs.end(), q.ordinal()) == devs.end()) devs.push_back(q.ordinal());
    return devs;
}
}
/// Sets the program header of q's device; this replaces the previous one until pop_program_header(q).
inline void push_program_header(const backend::command_queue &q, const std::string &str) {
    VEXB_CHECKED(vexb_program_header_push(q.ordinal(), str.c_str()));
}
/// Restores the program header q's device had before the last push.
inline void pop_program_header(const backend::command_queue &q) {
    VEXB_CHECKED(vexb_program_header_pop(q.ordinal()));
}
/// Sets the program header of every device of the queue list.
inline void push_program_header(const std::vector<backend::command_queue> &queue, const std::string &str) {
    for (int d : detail::header_devices(queue)) VEXB_CHECKED(vexb_program_header_push(d, str.c_str()));
}
/// Restores the previous program header of every device of the queue list.
inline void pop_program_header(const std::vector<backend::command_queue> &queue) {
    for (int d : detail::header_devices(queue)) VEXB_CHECKED(vexb_program_header_pop(d));
}
/// The effective program header of q's device ("" when none was pushed).
inline std::string get_program_header(const backend::command_queue &q) {
    size_t len = 0;
    VEXB_CHECKED(vexb_program_header_get(q.ordinal(), nullptr, &len));
    std::string h(len, '\0');
    VEXB_CHECKED(vexb_program_header_get(q.ordinal(), &h[0], &len));
    h.resize(len - 1);
    return h;
}
/// Pushes a program header on construction, pops it on destruction.
struct scoped_program_header {
    std::vector<backend::command_queue> q;
    scoped_program_header(const std::vector<backend::command_queue> &q, const std::string &str) : q(q) { push_program_header(this->q, str); }
    scoped_program_header(const backend::command_queue &q, const std::string &str) : q(1, q) { push_program_header(this->q, str); }
    ~scoped_program_header() { try { pop_program_header(q); } catch (...) {} }
    scoped_program_header(const scoped_program_header&) = delete;
    scoped_program_header& operator=(const scoped_program_header&) = delete;
};
}
#endif
