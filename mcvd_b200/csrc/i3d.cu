// Inception-v1 I3D features of videos for FVD: see MCVD_OP_I3D_PREP, MCVD_OP_CONV3D, MCVD_OP_MAXPOOL3D and
// MCVD_OP_I3D_HEAD in include/mcvd_b200.h.  One chunk of N videos is 72 launches whatever N is: prep, the stem and
// stage-2 convolutions (3), the stand-alone pools (4), 7 per Inception block (six convolutions and the b3a pool,
// 9 blocks) and the head.  The convolutions and pools are in conv_eval.cu.
#include "mcvd_common.cuh"

namespace mcvd {

constexpr int I3D_SIDE = 224;

// ------------------------------------------------------------------------------------------------
// prep: bilinear resize (ATen's align_corners=False source index), centre crop to 224x224, (x - 0.5) * 2; a grey
// frame is replicated to RGB and channel 3 is zero.  One thread per output pixel of one frame.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_i3d_prep(const float* __restrict__ src, float* __restrict__ dst, int C, int T,
                                                  int S, int Ht, int Wt) {
  const int pix = blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= I3D_SIDE * I3D_SIDE) return;
  const int frame = blockIdx.y;                    // video * T + t
  const int oy = pix / I3D_SIDE + (Ht - I3D_SIDE) / 2, ox = pix % I3D_SIDE + (Wt - I3D_SIDE) / 2;
  const float sh = (float)S / (float)Ht, sw = (float)S / (float)Wt;
  float fy = sh * ((float)oy + 0.5f) - 0.5f, fx = sw * ((float)ox + 0.5f) - 0.5f;
  fy = fy < 0.f ? 0.f : fy;
  fx = fx < 0.f ? 0.f : fx;
  const int y0 = (int)fy, x0 = (int)fx;
  const int y1 = y0 + (y0 < S - 1 ? 1 : 0), x1 = x0 + (x0 < S - 1 ? 1 : 0);
  const float ly1 = fy - (float)y0, lx1 = fx - (float)x0, ly0 = 1.f - ly1, lx0 = 1.f - lx1;
  const float* base = src + (long long)frame * C * S * S;   // [B, T*C, S, S]: frame-major, then channel
  float out[3] = {0.f, 0.f, 0.f};
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    if (c >= C) break;
    const float* p = base + (long long)c * S * S;
    const float v = ly0 * (lx0 * p[y0 * S + x0] + lx1 * p[y0 * S + x1]) +
                    ly1 * (lx0 * p[y1 * S + x0] + lx1 * p[y1 * S + x1]);
    out[c] = (v - 0.5f) * 2.0f;
  }
  float4 v;
  v.x = out[0];
  v.y = C == 1 ? out[0] : out[1];
  v.z = C == 1 ? out[0] : out[2];
  v.w = 0.0f;
  reinterpret_cast<float4*>(dst)[(long long)frame * I3D_SIDE * I3D_SIDE + pix] = v;
}

const char* i3d_prep_error(const McvdOp& op) {
  if (!op.src0 || !op.dst) return "null frames or output";
  if (op.C0 != 1 && op.C0 != 3) return "channels per frame must be 1 or 3";
  if (op.H != I3D_SIDE || op.W != I3D_SIDE) return "output side must be 224x224";
  if (op.i0 < 1 || op.i1 < 1) return "frames or input side out of range";
  if (op.i2 < I3D_SIDE || op.i3 < I3D_SIDE) return "resized size smaller than the 224x224 crop";
  if ((long long)op.B * op.i0 > 65535) return "too many frames for the grid";
  return nullptr;
}

int launch_i3d_prep(const McvdOp& op, cudaStream_t s) {
  if (const char* why = i3d_prep_error(op)) MCVD_CHECK(false, "I3D_PREP: %s", why);
  dim3 grid(cdiv(I3D_SIDE * I3D_SIDE, 256), (unsigned)(op.B * op.i0));
  k_i3d_prep<<<grid, 256, 0, s>>>((const float*)op.src0, (float*)op.dst, op.C0, op.i0, op.i1, op.i2, op.i3);
  MCVD_CUDA_LAUNCH_CHECK("i3d_prep");
  return 0;
}

// ------------------------------------------------------------------------------------------------
// head: AvgPool3d([2, 7, 7], stride 1) -> 1x1x1 logits conv with bias -> mean over time, fp64.  One CTA per video:
// per time window the block averages the 2*7*7 positions of every channel into shared memory (each channel by one
// thread, in a fixed order), then each thread takes its logits through the window's dot product in channel order.
// ------------------------------------------------------------------------------------------------
constexpr int HEAD_SIDE = 7;

__global__ void __launch_bounds__(256) k_i3d_head(const float* __restrict__ src, const float* __restrict__ w,
                                                  const float* __restrict__ bias, double* __restrict__ out, int T,
                                                  int C, int Cout) {
  extern __shared__ double avg[];
  const int vid = blockIdx.x;
  const float* x = src + (long long)vid * T * HEAD_SIDE * HEAD_SIDE * C;
  const int P = HEAD_SIDE * HEAD_SIDE;
  double acc[2] = {0.0, 0.0};                      // Cout <= 2 * blockDim.x
  for (int t = 0; t + 1 < T; ++t) {
    __syncthreads();                               // the previous window's dot products are done with avg
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
      double s = 0.0;
      for (int dt = 0; dt < 2; ++dt)
        for (int p = 0; p < P; ++p) s += (double)x[((long long)(t + dt) * P + p) * C + c];
      avg[c] = s / (double)(2 * P);
    }
    __syncthreads();
    for (int j = 0; j < 2; ++j) {
      const int o = threadIdx.x + j * blockDim.x;
      if (o >= Cout) break;
      double d = (double)bias[o];
      for (int c = 0; c < C; ++c) d += avg[c] * (double)w[(long long)c * Cout + o];
      acc[j] += d;
    }
  }
  for (int j = 0; j < 2; ++j) {
    const int o = threadIdx.x + j * blockDim.x;
    if (o < Cout) out[(long long)vid * Cout + o] = acc[j] / (double)(T - 1);
  }
}

const char* i3d_head_error(const McvdOp& op) {
  if (!op.src0 || !op.dst || !op.w || !op.bias) return "null features, output, weights or bias";
  if (op.i4 < 2) return "needs at least 2 time steps for the [2, 7, 7] average pool";
  if (op.i5 != HEAD_SIDE) return "input side must be 7 for the [2, 7, 7] average pool";
  if (op.C0 < 1 || op.C0 * (int)sizeof(double) > 48 * 1024) return "channels out of range (1 .. 6144)";
  if (op.Cout < 1 || op.Cout > 512) return "logits out of range (1 .. 512)";
  return nullptr;
}

int launch_i3d_head(const McvdOp& op, cudaStream_t s) {
  if (const char* why = i3d_head_error(op)) MCVD_CHECK(false, "I3D_HEAD: %s", why);
  k_i3d_head<<<op.B, 256, op.C0 * sizeof(double), s>>>((const float*)op.src0, (const float*)op.w,
                                                       (const float*)op.bias, (double*)op.dst, op.i4, op.C0, op.Cout);
  MCVD_CUDA_LAUNCH_CHECK("i3d_head");
  return 0;
}

}  // namespace mcvd
