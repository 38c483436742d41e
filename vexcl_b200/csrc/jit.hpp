// Run-time compilation helpers shared by the NVRTC side paths (csrc/jit.cu): expression kernels and the
// matrix-specialised CCSR kernel (csrc/ccsr.cu).
#pragma once
#include <string>
#include <cuda_runtime.h>

namespace vexb {
/// Compile `src` for sm_90a (--fmad=false) without touching a device; *cubin_bytes and *log are optional.
/// device_default adds --device-as-default-execution-space (programs with a user-function preamble).
int jit_compile_only(const std::string &src, size_t *cubin_bytes, std::string *log, bool device_default = false);
/// Compile `src`, load it on the CURRENT device and return the entry point `name`.  Cached by (source, options, device).
int jit_build(int dev, const std::string &src, const char *name, void **fn, bool device_default = false);
/// The effective program header of device `dev` (vexb_program_header_push), "" when none was pushed.
std::string program_header(int dev);
/// `src` with `header` at its very top (on a line of its own); `src` itself when the header is empty.
std::string with_program_header(const std::string &header, const std::string &src);
/// cuLaunchKernel on a function returned by jit_build.
int jit_launch(void *fn, unsigned grid, unsigned block, unsigned smem, cudaStream_t st, void **args);
}
