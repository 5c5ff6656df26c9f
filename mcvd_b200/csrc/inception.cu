// Inception-v3 pool features of frames for FID: see MCVD_OP_FID_PREP, MCVD_OP_CONV2D, MCVD_OP_MAXPOOL2D and
// MCVD_OP_FID_HEAD in include/mcvd_b200.h.  One chunk of N frames is 100 launches whatever N is: prep, the five stem
// convolutions and their two pools, every BasicConv2d of the eleven Inception blocks (the avg / max pools of the
// branch_pool convs are fused into their input read; the stride-2 pools of Mixed_6a and Mixed_7a are one launch
// each) and the head.  The convolutions and pools are in conv_eval.cu.
#include "mcvd_common.cuh"

namespace mcvd {

constexpr int FID_SIDE = 299;

// ------------------------------------------------------------------------------------------------
// prep: bilinear resize to 299x299 (ATen's align_corners=False source index and lambdas, no antialias), 2x - 1; a
// grey frame is replicated to RGB and channel 3 is zero.  One thread per output pixel of one frame.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_fid_prep(const float* __restrict__ src, float* __restrict__ dst, int C,
                                                  int S) {
  const int pix = blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= FID_SIDE * FID_SIDE) return;
  const int frame = blockIdx.y;
  const int oy = pix / FID_SIDE, ox = pix % FID_SIDE;
  const float scale = (float)S / (float)FID_SIDE;
  float fy = scale * ((float)oy + 0.5f) - 0.5f;
  float fx = scale * ((float)ox + 0.5f) - 0.5f;
  fy = fy < 0.f ? 0.f : fy;
  fx = fx < 0.f ? 0.f : fx;
  const int y0 = min((int)fy, S - 1), x0 = min((int)fx, S - 1);
  const int y1 = y0 + (y0 < S - 1 ? 1 : 0), x1 = x0 + (x0 < S - 1 ? 1 : 0);
  const float ly1 = fminf(fy - (float)y0, 1.f), lx1 = fminf(fx - (float)x0, 1.f);
  const float ly0 = 1.f - ly1, lx0 = 1.f - lx1;
  const float* base = src + (long long)frame * C * S * S;
  float out[3] = {0.f, 0.f, 0.f};
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    if (c >= C) break;
    const float* p = base + (long long)c * S * S;
    const float v = ly0 * (lx0 * p[y0 * S + x0] + lx1 * p[y0 * S + x1]) +
                    ly1 * (lx0 * p[y1 * S + x0] + lx1 * p[y1 * S + x1]);
    out[c] = 2.0f * v - 1.0f;                      // 2v is exact: one rounding, as the reference's 2 * x - 1
  }
  float4 v;
  v.x = out[0];
  v.y = C == 1 ? out[0] : out[1];
  v.z = C == 1 ? out[0] : out[2];
  v.w = 0.0f;
  reinterpret_cast<float4*>(dst)[(long long)frame * FID_SIDE * FID_SIDE + pix] = v;
}

const char* fid_prep_error(const McvdOp& op) {
  if (!op.src0 || !op.dst) return "null frames or output";
  if (op.C0 != 1 && op.C0 != 3) return "channels per frame must be 1 or 3";
  if (op.H != FID_SIDE || op.W != FID_SIDE) return "output side must be 299x299";
  if (op.i1 < 1) return "input side out of range";
  if (op.B > 65535) return "too many frames for the grid";
  return nullptr;
}

int launch_fid_prep(const McvdOp& op, cudaStream_t s) {
  if (const char* why = fid_prep_error(op)) MCVD_CHECK(false, "FID_PREP: %s", why);
  dim3 grid(cdiv(FID_SIDE * FID_SIDE, 256), (unsigned)op.B);
  k_fid_prep<<<grid, 256, 0, s>>>((const float*)op.src0, (float*)op.dst, op.C0, op.i1);
  MCVD_CUDA_LAUNCH_CHECK("fid_prep");
  return 0;
}

// ------------------------------------------------------------------------------------------------
// head: AdaptiveAvgPool2d(1) in fp64.  One thread per (frame, channel) sums the positions in raster order.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_fid_head(const float* __restrict__ src, double* __restrict__ out, int P,
                                                  int C, long long total) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const long long n = idx / C;
  const int c = (int)(idx - n * C);
  const float* x = src + n * P * C + c;
  double s = 0.0;
  for (int p = 0; p < P; ++p) s += (double)x[(long long)p * C];
  out[idx] = s / (double)P;
}

const char* fid_head_error(const McvdOp& op) {
  if (!op.src0 || !op.dst) return "null features or output";
  if (op.C0 < 1) return "channels out of range";
  if (op.i5 < 1) return "input side out of range";
  if (op.H != 1 || op.W != 1) return "output size must be 1x1";
  if (((long long)op.B * op.C0 + 255) / 256 > 0x7fffffffLL) return "too many outputs for the grid";
  return nullptr;
}

int launch_fid_head(const McvdOp& op, cudaStream_t s) {
  if (const char* why = fid_head_error(op)) MCVD_CHECK(false, "FID_HEAD: %s", why);
  const long long total = (long long)op.B * op.C0;
  k_fid_head<<<(unsigned)((total + 255) / 256), 256, 0, s>>>((const float*)op.src0, (double*)op.dst, op.i5 * op.i5,
                                                              op.C0, total);
  MCVD_CUDA_LAUNCH_CHECK("fid_head");
  return 0;
}

}  // namespace mcvd
