// Run-time compilation shared by every kernel NVRTC builds (csrc/jit.cu): expression, multi-expression and reduction
// kernels, the product kernel of user value types (csrc/bspmv.cu), stencil operators (csrc/stencil.cu) and the
// matrix-specialised CCSR kernel (csrc/ccsr.cu).  They all go through one program cache, jit_program.
#pragma once
#include <functional>
#include <string>
#include <cuda_runtime.h>

namespace vexb {
/// A program jit_program has not built yet, as its caller's source callback describes it.
struct JitBuild {
    long uses = 0;                  // in: requests of this program so far, this one included
    std::string text;               // out: the program without the header (jit_program puts the header on top)
    bool device_default = false;    // out: compile with --device-as-default-execution-space (programs with a preamble)
    bool background = false;        // out: compile on a background thread; the request gets no function
    bool later = false;             // out: do not compile yet; the request gets no function
};
using JitSource = std::function<int(JitBuild *)>;

/// The one cache of run-time compiled programs.  key: whatever determines the text apart from the header, distinct
/// between callers (each prefixes its own); name: the entry point; header: the device's program header in force for this
/// program ("" for none), which goes at the top of the text and into the key here and nowhere else.  On the first
/// request `source` runs on the calling thread; NVRTC then runs on this thread or, as `source` asks, on a background one,
/// holding no lock of the cache.  Returns the function loaded on device dev (the current device; dev < 0: compile only)
/// in *fn, or VEXB_OK with *fn = NULL when the program is not ready: delayed, compiling in the background, or compiling
/// on another thread while wait is false.  A failed compilation is remembered: every later request gets its status and
/// message.
int jit_program(int dev, const std::string &key, const char *name, const std::string &header, const JitSource &source,
                bool wait, void **fn);
/// The source printers' tail: with compile != 0, compile `src` for sm_90a without touching a device and append
/// "// NVRTC: ok, cubin N bytes" and the NVRTC log when it is not empty; then `src` into buf (*len in: capacity,
/// out: bytes needed; buf may be NULL).
int jit_print(std::string src, int compile, bool device_default, char *buf, size_t *len);
/// The effective program header of device `dev` (vexb_program_header_push), "" when none was pushed.
std::string program_header(int dev);
/// cuLaunchKernel on a function returned by jit_program.
int jit_launch(void *fn, unsigned grid, unsigned block, unsigned smem, cudaStream_t st, void **args);
}
