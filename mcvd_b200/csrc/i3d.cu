// Inception-v1 I3D features of videos for FVD: see MCVD_OP_I3D_PREP, MCVD_OP_CONV3D, MCVD_OP_MAXPOOL3D and
// MCVD_OP_I3D_HEAD in include/mcvd_b200.h.  One chunk of N videos is 72 launches whatever N is: prep, the stem and
// stage-2 convolutions (3), the stand-alone pools (4), 7 per Inception block (six convolutions and the b3a pool,
// 9 blocks) and the head.
#include <math.h>

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
// NDHWC 3-D convolution + bias + ReLU as an fp32 FFMA implicit GEMM: M = videos * To * So * So output positions,
// N = Cout, K = kt * ks * ks * Cin in (dt, dy, dx, c) order.  The tiling is k_conv_relu's (lpips.cu): 64 x 64 output
// tile per CTA, 16-deep K slices, 4 x 4 outputs per thread, the next slice prefetched into registers.  Cout only
// needs to be a multiple of 8 (n tiles are masked), and the result goes to channels [off, off + Cout) of a
// pitch-wide output, so an Inception block's branches write their concat in place.  Every output is accumulated by
// one thread in K order: a video's features do not depend on the batch or chunk it is computed in.
// PW: 1x1x1 stride-1 (most of I3D), where the output position is the input position.
// ------------------------------------------------------------------------------------------------
constexpr int C3_BM = 64, C3_BN = 64, C3_BK = 16;

struct Conv3Geom {
  int Tin, Sin, Cin, kt, ks, st, ss, pt, ps, To, So, Cout, K, pitch, off;
  long long M;
};

struct Gather3 {
  const float* vid;          // the position's video, NULL past the last position
  int it0, iy0, ix0;         // front-top-left input coordinate of its window
};

template <bool PW>
__device__ __forceinline__ Gather3 gather3_pos(const float* __restrict__ src, const Conv3Geom& g, long long m) {
  Gather3 q{nullptr, 0, 0, 0};
  if (m >= g.M) return q;
  if (PW) {
    q.vid = src + m * g.Cin;
    return q;
  }
  const int P = g.To * g.So * g.So;
  const long long n = m / P;
  int r = (int)(m - n * P);
  const int ot = r / (g.So * g.So);
  r -= ot * g.So * g.So;
  q.vid = src + n * g.Tin * g.Sin * g.Sin * g.Cin;
  q.it0 = ot * g.st - g.pt;
  q.iy0 = (r / g.So) * g.ss - g.ps;
  q.ix0 = (r % g.So) * g.ss - g.ps;
  return q;
}

template <bool PW>
__device__ __forceinline__ float4 conv3_gather(const Gather3& q, const Conv3Geom& g, int k) {
  const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
  if (!q.vid || k >= g.K) return zero;
  if (PW) return *reinterpret_cast<const float4*>(q.vid + k);
  const int tap = k / g.Cin, c = k - tap * g.Cin;
  const int kk = g.ks * g.ks;
  const int dt = tap / kk, r = tap - dt * kk;
  const int dy = r / g.ks;
  const int it = q.it0 + dt, iy = q.iy0 + dy, ix = q.ix0 + r - dy * g.ks;
  if (it < 0 || it >= g.Tin || iy < 0 || iy >= g.Sin || ix < 0 || ix >= g.Sin) return zero;
  return *reinterpret_cast<const float4*>(q.vid + (((long long)it * g.Sin + iy) * g.Sin + ix) * g.Cin + c);
}

template <bool PW>
__global__ void __launch_bounds__(256, 4) k_conv3d(const float* __restrict__ src, const float* __restrict__ w,
                                                const float* __restrict__ bias, float* __restrict__ dst, Conv3Geom g) {
  __shared__ __align__(16) float As[2][C3_BK][C3_BM];
  __shared__ __align__(16) float Bs[2][C3_BK][C3_BN];
  const int tid = threadIdx.x;
  const long long m0 = (long long)blockIdx.x * C3_BM;
  const int n0 = blockIdx.y * C3_BN;
  const int am = tid % C3_BM, ak = (tid / C3_BM) * 4;
  const int bk = tid / (C3_BN / 4), bn = (tid % (C3_BN / 4)) * 4;
  const int tm = (tid / 16) * 4, tn = (tid % 16) * 4;
  const bool bcol = n0 + bn < g.Cout;             // Cout % 8 == 0: a 4-channel group is wholly in or out
  float acc[4][4] = {};
  const Gather3 q = gather3_pos<PW>(src, g, m0 + am);
  float4 ra = conv3_gather<PW>(q, g, ak);
  float4 rb = bcol && bk < g.K ? *reinterpret_cast<const float4*>(w + (long long)bk * g.Cout + n0 + bn)
                               : make_float4(0.f, 0.f, 0.f, 0.f);
  int buf = 0;
  for (int k0 = 0; k0 < g.K; k0 += C3_BK) {
    As[buf][ak + 0][am] = ra.x; As[buf][ak + 1][am] = ra.y; As[buf][ak + 2][am] = ra.z; As[buf][ak + 3][am] = ra.w;
    *reinterpret_cast<float4*>(&Bs[buf][bk][bn]) = rb;
    __syncthreads();
    const int k1 = k0 + C3_BK;
    if (k1 < g.K) {
      ra = conv3_gather<PW>(q, g, k1 + ak);
      rb = bcol && k1 + bk < g.K ? *reinterpret_cast<const float4*>(w + (long long)(k1 + bk) * g.Cout + n0 + bn)
                                 : make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll
    for (int kk = 0; kk < C3_BK; ++kk) {
      const float4 a = *reinterpret_cast<const float4*>(&As[buf][kk][tm]);
      const float4 b = *reinterpret_cast<const float4*>(&Bs[buf][kk][tn]);
      const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    buf ^= 1;                                      // the other buffer was last read before this slice's barrier
  }
  if (n0 + tn >= g.Cout) return;
  const float4 bb = *reinterpret_cast<const float4*>(bias + n0 + tn);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const long long m = m0 + tm + i;
    if (m >= g.M) break;
    float4 o;
    o.x = fmaxf(acc[i][0] + bb.x, 0.f);
    o.y = fmaxf(acc[i][1] + bb.y, 0.f);
    o.z = fmaxf(acc[i][2] + bb.z, 0.f);
    o.w = fmaxf(acc[i][3] + bb.w, 0.f);
    *reinterpret_cast<float4*>(dst + m * g.pitch + g.off + n0 + tn) = o;
  }
}

const char* conv3d_error(const McvdOp& op) {
  if (!op.src0 || !op.dst || !op.w || !op.bias) return "null input, output, weights or bias";
  if (op.C0 <= 0 || op.C0 % 4) return "input channels must be a positive multiple of 4";
  if (op.Cout <= 0 || op.Cout % 8) return "output channels must be a positive multiple of 8";
  if (op.i0 < 1 || op.i1 < 1 || op.i2 < 1 || op.i3 < 1) return "kernel size or stride out of range";
  if (op.i4 < 1 || op.i5 < 1) return "input size out of range";
  if (op.i7 < 0 || op.i7 % 4 || op.i6 % 4 || op.i6 < op.i7 + op.Cout)
    return "channel pitch must be a multiple of 4 and at least offset + Cout (offset a multiple of 4)";
  if (op.H != op.W || op.H != same_out(op.i5, op.i1, op.i3)) return "output size disagrees with the SAME geometry";
  const long long K = (long long)op.i0 * op.i1 * op.i1 * op.C0;
  if (K > (1LL << 30)) return "reduction too long";
  const long long M = (long long)op.B * same_out(op.i4, op.i0, op.i2) * op.H * op.W;
  if ((M + C3_BM - 1) / C3_BM > 0x7fffffffLL) return "too many output positions for the grid";
  return nullptr;
}

int launch_conv3d(const McvdOp& op, cudaStream_t s) {
  if (const char* why = conv3d_error(op)) MCVD_CHECK(false, "CONV3D: %s", why);
  Conv3Geom g;
  g.Tin = op.i4; g.Sin = op.i5; g.Cin = op.C0; g.kt = op.i0; g.ks = op.i1; g.st = op.i2; g.ss = op.i3;
  g.pt = same_pad(op.i4, op.i0, op.i2) / 2;
  g.ps = same_pad(op.i5, op.i1, op.i3) / 2;
  g.To = same_out(op.i4, op.i0, op.i2); g.So = op.H;
  g.Cout = op.Cout; g.K = op.i0 * op.i1 * op.i1 * op.C0; g.pitch = op.i6; g.off = op.i7;
  g.M = (long long)op.B * g.To * g.So * g.So;
  dim3 grid((unsigned)((g.M + C3_BM - 1) / C3_BM), (unsigned)cdiv(op.Cout, C3_BN));
  const bool pw = op.i0 == 1 && op.i1 == 1 && op.i2 == 1 && op.i3 == 1;
  if (pw) k_conv3d<true><<<grid, 256, 0, s>>>((const float*)op.src0, (const float*)op.w, (const float*)op.bias,
                                               (float*)op.dst, g);
  else k_conv3d<false><<<grid, 256, 0, s>>>((const float*)op.src0, (const float*)op.w, (const float*)op.bias,
                                            (float*)op.dst, g);
  MCVD_CUDA_LAUNCH_CHECK("conv3d");
  return 0;
}

// ------------------------------------------------------------------------------------------------
// SAME max-pool with zero padding (MaxPool3dSamePadding: F.pad with zeros, then nn.MaxPool3d).  One thread per
// output position and 4-channel group.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_maxpool3d(const float* __restrict__ src, float* __restrict__ dst, int Tin,
                                                   int Sin, int C4, int kt, int ks, int st, int ss, int pt, int ps,
                                                   int To, int So, long long total) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int c4 = (int)(idx % C4);
  long long r = idx / C4;
  const int ox = (int)(r % So); r /= So;
  const int oy = (int)(r % So); r /= So;
  const int ot = (int)(r % To);
  const long long n = r / To;
  const float4* vid = reinterpret_cast<const float4*>(src) + n * Tin * Sin * Sin * C4 + c4;
  const int t0 = ot * st - pt, y0 = oy * ss - ps, x0 = ox * ss - ps;
  float4 v = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
  for (int dt = 0; dt < kt; ++dt)
    for (int dy = 0; dy < ks; ++dy)
      for (int dx = 0; dx < ks; ++dx) {
        const int it = t0 + dt, iy = y0 + dy, ix = x0 + dx;
        float4 u = make_float4(0.f, 0.f, 0.f, 0.f);  // the zero padding takes part in the max
        if (it >= 0 && it < Tin && iy >= 0 && iy < Sin && ix >= 0 && ix < Sin)
          u = vid[(((long long)it * Sin + iy) * Sin + ix) * C4];
        v.x = fmaxf(v.x, u.x); v.y = fmaxf(v.y, u.y); v.z = fmaxf(v.z, u.z); v.w = fmaxf(v.w, u.w);
      }
  reinterpret_cast<float4*>(dst)[idx] = v;
}

const char* maxpool3d_error(const McvdOp& op) {
  if (!op.src0 || !op.dst) return "null input or output";
  if (op.C0 <= 0 || op.C0 % 4) return "channels must be a positive multiple of 4";
  if (op.i0 < 1 || op.i1 < 1 || op.i2 < 1 || op.i3 < 1) return "window or stride out of range";
  if (op.i4 < 1 || op.i5 < 1) return "input size out of range";
  if (op.H != op.W || op.H != same_out(op.i5, op.i1, op.i3)) return "output size disagrees with the SAME geometry";
  const long long total = (long long)op.B * same_out(op.i4, op.i0, op.i2) * op.H * op.W * (op.C0 / 4);
  if ((total + 255) / 256 > 0x7fffffffLL) return "too many outputs for the grid";
  return nullptr;
}

int launch_maxpool3d(const McvdOp& op, cudaStream_t s) {
  if (const char* why = maxpool3d_error(op)) MCVD_CHECK(false, "MAXPOOL3D: %s", why);
  const int To = same_out(op.i4, op.i0, op.i2);
  const long long total = (long long)op.B * To * op.H * op.W * (op.C0 / 4);
  k_maxpool3d<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(
      (const float*)op.src0, (float*)op.dst, op.i4, op.i5, op.C0 / 4, op.i0, op.i1, op.i2, op.i3,
      same_pad(op.i4, op.i0, op.i2) / 2, same_pad(op.i5, op.i1, op.i3) / 2, To, op.H, total);
  MCVD_CUDA_LAUNCH_CHECK("maxpool3d");
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
