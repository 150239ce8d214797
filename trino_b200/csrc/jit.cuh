// jit.cuh — NVRTC specialisation service (see jit.cu)
#pragma once
#include <string>

#include "common.cuh"

namespace tg {

bool jit_available();
const char* jit_unavailable_reason();
// compile device_lib.cuh + body for sm_90a and return the cubin (works without a GPU)
int jit_compile_cubin(tgpu_ctx* ctx, const std::string& body, std::string* cubin);
// compiled + loaded + cached kernel handle (CUfunction) for the current device
int jit_get_function(tgpu_ctx* ctx, const std::string& body, const char* kernel_name, void** fn_out);
// CTAs of this kernel that fit one SM (grid-stride kernels are launched as exactly one resident wave)
int jit_blocks_per_sm(void* fn, int block, size_t smem);
int jit_launch(tgpu_ctx* ctx, void* fn, int grid, int block, size_t smem, void** params);

}  // namespace tg
