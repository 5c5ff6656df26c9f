// Shared helpers for the mcvd_b200 kernels (sm_90a).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/mcvd_b200.h"

namespace mcvd {

void set_error(const char* fmt, ...);

#define MCVD_CHECK(cond, ...)                   \
  do {                                          \
    if (!(cond)) {                              \
      ::mcvd::set_error(__VA_ARGS__);           \
      return -1;                                \
    }                                           \
  } while (0)

#define MCVD_CUDA_LAUNCH_CHECK(name)                                              \
  do {                                                                            \
    cudaError_t e__ = cudaGetLastError();                                         \
    if (e__ != cudaSuccess) {                                                     \
      ::mcvd::set_error("%s: launch failed: %s", name, cudaGetErrorString(e__)); \
      return -2;                                                                  \
    }                                                                             \
  } while (0)

__host__ __device__ inline int cdiv(int a, int b) { return (a + b - 1) / b; }

__device__ __forceinline__ float silu_f(float v) { return v / (1.0f + expf(-v)); }

// launchers (one per op kind); each returns 0 or a negative error code
int launch_nchw_to_nhwc(const McvdOp& op, cudaStream_t s);
int launch_nhwc_to_nchw(const McvdOp& op, cudaStream_t s);
int launch_timestep_embed(const McvdOp& op, cudaStream_t s);
int launch_linear(const McvdOp& op, cudaStream_t s);
int launch_gn_partial(const McvdOp& op, cudaStream_t s);
int launch_gn_finalize(const McvdOp& op, cudaStream_t s);
int launch_apply(const McvdOp& op, cudaStream_t s);
int launch_conv_simt(const McvdOp& op, cudaStream_t s);
int launch_attention(const McvdOp& op, cudaStream_t s);
int launch_resize_nearest(const McvdOp& op, cudaStream_t s);
int launch_diffusion_update(const McvdOp& op, cudaStream_t s);
int launch_conv_umma(const McvdOp& op, cudaStream_t s);
int launch_conv_umma2(const McvdOp& op, cudaStream_t s);
int launch_conv_smalln(const McvdOp& op, cudaStream_t s);
int launch_copy(const McvdOp& op, cudaStream_t s);
int launch_attention_umma(const McvdOp& op, cudaStream_t s);
int launch_frame_metrics(const McvdOp& op, cudaStream_t s);

}  // namespace mcvd
