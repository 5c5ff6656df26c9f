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

// TF-"SAME" padding of one axis (pytorch_i3d.py compute_pad): the total; the front gets total / 2
__host__ __device__ inline int same_pad(int in, int k, int s) {
  const int r = in % s;
  const int p = r == 0 ? k - s : k - r;
  return p > 0 ? p : 0;
}

// output extent of one axis after SAME padding: (in + pad - k) / s + 1, which is ceil(in / s) for I3D's shapes
__host__ __device__ inline int same_out(int in, int k, int s) { return (in + same_pad(in, k, s) - k) / s + 1; }

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
// key tile the attention kernels run T tokens at head dim d with; 0 where they are not built for the shape
int attention_simt_key_tile(int T, int d);
int attention_umma_key_tile(int T, int d);
int launch_frame_metrics(const McvdOp& op, cudaStream_t s);
int launch_noise(const McvdOp& op, cudaStream_t s);
int launch_lpips_prep(const McvdOp& op, cudaStream_t s);
int launch_lpips_layer(const McvdOp& op, cudaStream_t s);
int launch_i3d_prep(const McvdOp& op, cudaStream_t s);
int launch_i3d_head(const McvdOp& op, cudaStream_t s);
int launch_dsm_perturb(const McvdOp& op, cudaStream_t s);
int launch_dsm_loss(const McvdOp& op, cudaStream_t s);
int launch_fid_prep(const McvdOp& op, cudaStream_t s);
int launch_fid_head(const McvdOp& op, cudaStream_t s);
int launch_knn(const McvdOp& op, cudaStream_t s);
int launch_conv_ffma(const McvdOp& op, cudaStream_t s);   // CONV_RELU, CONV3D, CONV2D (conv_eval.cu)
int launch_maxpool(const McvdOp& op, cudaStream_t s);     // MAXPOOL3D, MAXPOOL2D (conv_eval.cu)
int launch_conv_tf32(const McvdOp& op, cudaStream_t s);   // CONV3D_TF32, CONV2D_TF32, CONV_RELU_TF32 (conv_tf32.cu)

// NULL, or why an op of the I3D kinds is unusable (shared by validation and launch; i3d.cu)
const char* i3d_prep_error(const McvdOp& op);
const char* i3d_head_error(const McvdOp& op);

// NULL, or why a MCVD_OP_DSM_PERTURB / MCVD_OP_DSM_LOSS op is unusable (shared by validation and launch; dsm.cu)
const char* dsm_error(const McvdOp& op);

// NULL, or why an op of the FID kinds is unusable (shared by validation and launch; inception.cu, knn.cu).  The conv
// and max-pool kinds of LPIPS, I3D and Inception-v3 are validated by conv_geom / conv_tf32_geom (conv_eval.cuh).
const char* fid_prep_error(const McvdOp& op);
const char* fid_head_error(const McvdOp& op);
const char* knn_error(const McvdOp& op);

// NULL, or why the Gamma parameters (f6 = shape, f7 = scale) of an op with MCVD_F_GAMMA are unusable
const char* gamma_params_error(const McvdOp& op);

}  // namespace mcvd
