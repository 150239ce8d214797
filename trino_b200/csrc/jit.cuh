// jit.cuh — NVRTC specialisation service (see jit.cu)
#pragma once
#include <functional>
#include <string>

#include "common.cuh"

namespace tg {

bool jit_available();
const char* jit_unavailable_reason();
// compile device_lib.cuh + body for sm_90a and return the cubin (works without a GPU)
int jit_compile_cubin(tgpu_ctx* ctx, const std::string& body, std::string* cubin);
// the tgpu_jit_selftest_* test hooks (no GPU needed): `gen` writes the source for the element sizes of the channel types; the source
// goes to source_out and is compiled, and *cubin_bytes gets the cubin's size, or source_out the compiler's error
int jit_selftest(const int32_t* channel_types, int32_t num_channels, const std::function<std::string(const int* elems)>& gen, int64_t* cubin_bytes,
                 char* source_out, int64_t source_cap);
// compiled + loaded + cached kernel handle (CUfunction) for the current device
int jit_get_function(tgpu_ctx* ctx, const std::string& body, const char* kernel_name, void** fn_out);
// CTAs of this kernel that fit one SM (grid-stride kernels are launched as exactly one resident wave)
int jit_blocks_per_sm(void* fn, int block, size_t smem);
int jit_launch(tgpu_ctx* ctx, void* fn, int grid, int block, size_t smem, void** params);

}  // namespace tg
