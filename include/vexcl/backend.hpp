#ifndef VEXCL_BACKEND_HPP
#define VEXCL_BACKEND_HPP
/*
 * vex::backend for the H100 build: thin RAII shells over the C ABI of
 * libvexb200.so (include/vexb200.h).  The names follow the reference's CUDA
 * flavour of the backend layer so that code written against it keeps compiling:
 *   device, command_queue, device_vector<T>, error, mem flags, duplicate_queue,
 *   is_cpu, queue_list            (vexcl/backend/cuda/context.hpp:96-413,
 *                                  vexcl/backend/cuda/device_vector.hpp:42-210,
 *                                  vexcl/backend/cuda/error.hpp:49-160)
 * There is no kernel / build_sources here: kernels are pre-compiled sm_90a
 * code inside the library, selected at run time from an expression IR (see
 * operations.hpp).  source_generator is reduced to what the snippets of a
 * user's vex::sparse::spmv_ops_impl need (sparse/spmv_ops.hpp).
 */
#include <cstddef>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <iostream>
#include <memory>
#include <sstream>
#include <stdexcept>
#include <string>
#include <vector>

#include "../vexb200.h"

namespace vex {
namespace backend {

/// All failures of the back end surface as this exception (file:line + message of the C ABI).
class error : public std::runtime_error {
    public:
        error(int code, const std::string &msg) : std::runtime_error(msg), code_(code) {}
        int code() const { return code_; }
    private:
        int code_;
};

inline std::ostream& operator<<(std::ostream &os, const error &e) {
    return os << "vexb error " << e.code() << ": " << e.what();
}

inline void check(int status, const char *file, int line) {
    if (status != VEXB_OK) {
        std::ostringstream msg;
        msg << file << ":" << line << "\n\t" << vexb_last_error();
        throw error(status, msg.str());
    }
}
#define VEXB_CHECKED(call) ::vex::backend::check((call), __FILE__, __LINE__)

typedef unsigned mem_flags;
static const mem_flags MEM_READ_ONLY  = 1;
static const mem_flags MEM_WRITE_ONLY = 2;
static const mem_flags MEM_READ_WRITE = 4;

/// A CUDA device ordinal with its properties.
class device {
    public:
        device(int ordinal = 0) : d(ordinal) {}
        int raw() const { return d; }
        std::string name() const { return props().name; }
        std::pair<int,int> compute_capability() const { auto p = props(); return std::make_pair(p.cc_major, p.cc_minor); }
        size_t multiprocessor_count() const { return props().sm_count; }
        size_t max_threads_per_block() const { return props().max_threads_per_block; }
        size_t max_shared_memory_per_block() const { return props().smem_per_block_optin; }
        size_t warp_size() const { return props().warp_size; }
        size_t global_mem_size() const { return props().total_mem; }
        bool operator==(const device &o) const { return d == o.d; }
    private:
        int d;
        vexb_devprops props() const { vexb_devprops p; VEXB_CHECKED(vexb_device_props(d, &p)); return p; }
};

/// The primary context of a device (kept for source compatibility; carries no state).
class context {
    public:
        context(device dev = device()) : dev(dev) {}
        int raw() const { return dev.raw(); }
        void set_current() const {}
        device get_device() const { return dev; }
        bool operator==(const context &o) const { return dev == o.dev; }
    private:
        device dev;
};

/// A stream on a device.  Copies share the stream.
class command_queue {
    public:
        command_queue() : dev(0) {}
        explicit command_queue(vex::backend::device d, unsigned flags = 0) : dev(d), f(flags) {
            void *s = nullptr;
            VEXB_CHECKED(vexb_stream_create(d.raw(), &s));
            int ord = d.raw();
            strm.reset(s, [ord](void *p) { vexb_stream_destroy(ord, p); });
        }
        command_queue(const vex::backend::context &c, vex::backend::device d, unsigned flags = 0) : command_queue(d, flags) { (void)c; }

        void finish() const { VEXB_CHECKED(vexb_stream_sync(dev.raw(), strm.get())); }
        vex::backend::device  device()  const { return dev; }
        vex::backend::context context() const { return vex::backend::context(dev); }
        unsigned flags() const { return f; }
        void* raw() const { return strm.get(); }
        int ordinal() const { return dev.raw(); }
        bool operator==(const command_queue &o) const { return strm.get() == o.strm.get(); }
        bool operator<(const command_queue &o) const { return strm.get() < o.strm.get(); }
    private:
        vex::backend::device dev;
        unsigned f = 0;
        std::shared_ptr<void> strm;
};

typedef int device_id;
typedef int context_id;
inline void select_context(const command_queue&) {}
inline device  get_device(const command_queue &q)     { return q.device(); }
inline device_id get_device_id(const command_queue &q)  { return q.ordinal(); }
inline context_id get_context_id(const command_queue &q) { return q.ordinal(); }
inline context get_context(const command_queue &q)    { return q.context(); }
inline command_queue duplicate_queue(const command_queue &q) { return command_queue(q.device(), q.flags()); }
inline bool is_cpu(const command_queue&) { return false; }

/// Device memory.  Copies alias the same allocation (as the reference's device_vector does).
template <typename T>
class device_vector {
    public:
        typedef T value_type;

        device_vector() : n(0), dev(0) {}

        device_vector(const command_queue &q, size_t n) : n(n), dev(q.ordinal()) { alloc(); }

        template <typename H>
        device_vector(const command_queue &q, size_t n, const H *host = 0, mem_flags = MEM_READ_WRITE)
            : n(n), dev(q.ordinal())
        {
            alloc();
            if (host && n) {
                if (std::is_same<T, H>::value) {
                    write(q, 0, n, reinterpret_cast<const T*>(host), true);
                } else {
                    std::vector<T> tmp(host, host + n);
                    write(q, 0, n, tmp.data(), true);
                }
            }
        }

        void write(const command_queue &q, size_t offset, size_t size, const T *host, bool blocking = false) const {
            if (size) VEXB_CHECKED(vexb_h2d(dev, raw_ptr() + offset, host, size * sizeof(T), q.raw(), blocking));
        }
        void read(const command_queue &q, size_t offset, size_t size, T *host, bool blocking = false) const {
            if (size) VEXB_CHECKED(vexb_d2h(dev, host, raw_ptr() + offset, size * sizeof(T), q.raw(), blocking));
        }

        size_t size() const { return n; }
        T* raw_ptr() const { return static_cast<T*>(buf.get()); }
        void* raw() const { return buf.get(); }
        int ordinal() const { return dev; }

        template <typename U>
        device_vector<U> reinterpret() const {
            device_vector<U> r; r.assign_raw(buf, n * sizeof(T) / sizeof(U), dev); return r;
        }
        void assign_raw(std::shared_ptr<void> b, size_t count, int d) { buf = b; n = count; dev = d; }

        /// Host view: copied out on creation, copied back on release.
        struct unmapper {
            device_vector<T> owner; command_queue q; size_t n;
            void operator()(T *p) const { if (p) { owner.write(q, 0, n, p, true); delete[] p; } }
        };
        typedef std::unique_ptr<T[], unmapper> mapped_array;

        mapped_array map(const command_queue &q) {
            T *p = new T[n ? n : 1];
            read(q, 0, n, p, true);
            return mapped_array(p, unmapper{*this, q, n});
        }
        mapped_array map(const command_queue &q) const { return const_cast<device_vector*>(this)->map(q); }
    private:
        size_t n;
        int dev;
        std::shared_ptr<void> buf;

        void alloc() {
            void *p = nullptr;
            VEXB_CHECKED(vexb_malloc(dev, n * sizeof(T), &p));
            int d = dev;
            buf.reset(p, [d](void *q) { vexb_free(d, q); });
        }
};

} // namespace backend

typedef backend::error error;

/// Device filters (vexcl/devlist.hpp:53-223, vexcl/backend/cuda/filter.hpp:46-106).
namespace Filter {

typedef std::function<bool(const backend::device&)> predicate;

struct General {
    predicate fn;
    General() : fn([](const backend::device&) { return true; }) {}
    template <class F> General(F f) : fn(f) {}
    bool operator()(const backend::device &d) const { return fn(d); }
};

inline General operator&&(General a, General b) { return General([a, b](const backend::device &d) { return a(d) && b(d); }); }
inline General operator||(General a, General b) { return General([a, b](const backend::device &d) { return a(d) || b(d); }); }
inline General operator!(General a) { return General([a](const backend::device &d) { return !a(d); }); }

static const General Any;
static const General All;
static const General GPU;
static const General DoublePrecision;
static const General CPU        = General([](const backend::device&) { return false; });
static const General Accelerator = General([](const backend::device&) { return false; });

/// First n devices that reach this filter (stateful; put it last in a conjunction).
inline General Count(int n) {
    auto left = std::make_shared<int>(n);
    return General([left](const backend::device&) { return (*left)-- > 0; });
}
/// The device at position n among those that reach this filter.
inline General Position(int n) {
    auto pos = std::make_shared<int>(0);
    return General([pos, n](const backend::device&) { return (*pos)++ == n; });
}
inline General Name(std::string s) {
    return General([s](const backend::device &d) { return d.name().find(s) != std::string::npos; });
}
inline General CC(int major, int minor) {
    return General([major, minor](const backend::device &d) { return d.compute_capability() >= std::make_pair(major, minor); });
}
template <class F> inline General Exclusive(F f) { return General(f); }

/// Environment filter: OCL_DEVICE (name substring), OCL_MAX_DEVICES, OCL_POSITION.
inline General make_env() {
    General f;
    if (const char *name = std::getenv("OCL_DEVICE")) f = f && Name(name);
    if (const char *maxdev = std::getenv("OCL_MAX_DEVICES")) f = f && Count(std::atoi(maxdev));
    if (const char *pos = std::getenv("OCL_POSITION")) f = f && Position(std::atoi(pos));
    return f;
}
struct EnvFilter {
    operator General() const { return make_env(); }
    bool operator()(const backend::device &d) const { return make_env()(d); }
};
static const EnvFilter Env;
inline General operator&&(EnvFilter, General b) { return make_env() && b; }
inline General operator&&(General a, EnvFilter) { return a && make_env(); }
inline General operator&&(EnvFilter, EnvFilter) { return make_env(); }

} // namespace Filter

namespace backend {

/// Devices passing the filter, each with one fresh stream (cuda/context.hpp:385-413).
template <class DevFilter>
std::pair<std::vector<context>, std::vector<command_queue>> queue_list(DevFilter &&filter, unsigned queue_flags = 0) {
    VEXB_CHECKED(vexb_init());
    int n = 0;
    VEXB_CHECKED(vexb_device_count(&n));
    Filter::General f = filter;
    std::vector<context> ctx;
    std::vector<command_queue> queue;
    for (int d = 0; d < n; ++d) {
        device dev(d);
        if (!f(dev)) continue;
        ctx.push_back(context(dev));
        queue.push_back(command_queue(dev, queue_flags));
    }
    return std::make_pair(ctx, queue);
}

template <class DevFilter>
std::vector<device> device_list(DevFilter &&filter) {
    VEXB_CHECKED(vexb_init());
    int n = 0;
    VEXB_CHECKED(vexb_device_count(&n));
    Filter::General f = filter;
    std::vector<device> out;
    for (int d = 0; d < n; ++d) if (f(device(d))) out.push_back(device(d));
    return out;
}

/// The part of the reference's source generator (vexcl/backend/cuda/source.hpp) that vex::sparse::spmv_ops_impl bodies
/// use: they write the device snippets of a user value type's sparse product (sparse/spmv_ops.hpp).  Numbers are written
/// with enough digits to read back the same double.
class source_generator {
    public:
        source_generator() { src.precision(17); }
        source_generator& new_line() { src << "\n" << std::string(2 * indent, ' '); return *this; }
        source_generator& open(const char *bracket) { new_line() << bracket; ++indent; return *this; }
        source_generator& close(const char *bracket) { if (indent) --indent; new_line() << bracket; return *this; }
        template <class T> source_generator& operator<<(const T &v) { src << v; return *this; }
        std::string str() const { return src.str(); }
    private:
        std::ostringstream src;
        unsigned indent = 2;            // the snippets go into the body of a loop of the generated kernel
};

} // namespace backend
} // namespace vex

#endif
