// Inception-v3 pool features of frames for FID: see MCVD_OP_FID_PREP, MCVD_OP_CONV2D, MCVD_OP_MAXPOOL2D and
// MCVD_OP_FID_HEAD in include/mcvd_b200.h.  One chunk of N frames is 100 launches whatever N is: prep, the five stem
// convolutions and their two pools, every BasicConv2d of the eleven Inception blocks (the avg / max pools of the
// branch_pool convs are fused into their input read; the stride-2 pools of Mixed_6a and Mixed_7a are one launch
// each) and the head.
#include <math.h>

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
// BasicConv2d (conv without bias, folded BatchNorm, ReLU) as an NHWC fp32 FFMA implicit GEMM: M = frames * Ho * Wo
// output positions, N = Cout, K = kh * kw * Cin in (dy, dx, c) order.  The tiling is k_conv3d's (i3d.cu): 64 x 64
// output tile per CTA, 16-deep K slices, 4 x 4 outputs per thread, the next slice prefetched into registers.  The
// result goes to channels [off, off + Cout) of a pitch-wide output, so an Inception block's branches write their
// concat in place.  Every output is accumulated by one thread in K order: a frame's features do not depend on the
// batch or chunk it is computed in.
// Gather modes: GENERAL (any kernel, stride, padding), PW (1x1, stride 1, no padding: the output position is the
// input position), and PW with the 3x3 / stride-1 / pad-1 pool of the branch_pool convs applied on the read: MAX
// (padding never wins) or AVG (count_include_pad=False: the sum of the taps inside the map over their number).
// ------------------------------------------------------------------------------------------------
constexpr int FC_BM = 64, FC_BN = 64, FC_BK = 16;
enum { G_GENERAL = 0, G_PW = 1, G_MAXPOOL = 2, G_AVGPOOL = 3 };

struct Conv2Geom {
  int Sin, Cin, kh, kw, stride, ph, pw, Ho, Wo, Cout, K, pitch, off;
  long long M;
};

struct Gather2 {
  const float* img;          // the position's frame (its input pixel for PW), NULL past the last position
  int iy0, ix0;              // top-left input coordinate of its window (the position itself for the pools)
};

template <int MODE>
__device__ __forceinline__ Gather2 gather2_pos(const float* __restrict__ src, const Conv2Geom& g, long long m) {
  Gather2 q{nullptr, 0, 0};
  if (m >= g.M) return q;
  if (MODE == G_PW) {
    q.img = src + m * g.Cin;
    return q;
  }
  const int P = g.Ho * g.Wo;
  const long long n = m / P;
  const int r = (int)(m - n * P);
  q.img = src + n * g.Sin * g.Sin * g.Cin;
  q.iy0 = (r / g.Wo) * g.stride - g.ph;
  q.ix0 = (r % g.Wo) * g.stride - g.pw;
  return q;
}

template <int MODE>
__device__ __forceinline__ float4 conv2_gather(const Gather2& q, const Conv2Geom& g, int k) {
  const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
  if (!q.img || k >= g.K) return zero;
  if (MODE == G_PW) return *reinterpret_cast<const float4*>(q.img + k);
  if (MODE == G_GENERAL) {
    const int tap = k / g.Cin, c = k - tap * g.Cin;
    const int dy = tap / g.kw;
    const int iy = q.iy0 + dy, ix = q.ix0 + tap - dy * g.kw;
    if (iy < 0 || iy >= g.Sin || ix < 0 || ix >= g.Sin) return zero;
    return *reinterpret_cast<const float4*>(q.img + ((long long)iy * g.Sin + ix) * g.Cin + c);
  }
  const float init = MODE == G_MAXPOOL ? -INFINITY : 0.f;
  float4 v = make_float4(init, init, init, init);
  int count = 0;
  for (int dy = -1; dy <= 1; ++dy)
    for (int dx = -1; dx <= 1; ++dx) {
      const int iy = q.iy0 + dy, ix = q.ix0 + dx;
      if (iy < 0 || iy >= g.Sin || ix < 0 || ix >= g.Sin) continue;
      const float4 u = *reinterpret_cast<const float4*>(q.img + ((long long)iy * g.Sin + ix) * g.Cin + k);
      if (MODE == G_MAXPOOL) {
        v.x = fmaxf(v.x, u.x); v.y = fmaxf(v.y, u.y); v.z = fmaxf(v.z, u.z); v.w = fmaxf(v.w, u.w);
      } else {
        v.x += u.x; v.y += u.y; v.z += u.z; v.w += u.w;
        ++count;
      }
    }
  if (MODE == G_AVGPOOL) {
    const float d = (float)count;
    v.x /= d; v.y /= d; v.z /= d; v.w /= d;
  }
  return v;
}

template <int MODE>
__global__ void __launch_bounds__(256, MODE >= G_MAXPOOL ? 2 : 4)
    k_conv2d(const float* __restrict__ src, const float* __restrict__ w, const float* __restrict__ bias,
             float* __restrict__ dst, Conv2Geom g) {
  __shared__ __align__(16) float As[2][FC_BK][FC_BM];
  __shared__ __align__(16) float Bs[2][FC_BK][FC_BN];
  const int tid = threadIdx.x;
  const long long m0 = (long long)blockIdx.x * FC_BM;
  const int n0 = blockIdx.y * FC_BN;
  const int am = tid % FC_BM, ak = (tid / FC_BM) * 4;
  const int bk = tid / (FC_BN / 4), bn = (tid % (FC_BN / 4)) * 4;
  const int tm = (tid / 16) * 4, tn = (tid % 16) * 4;
  const bool bcol = n0 + bn < g.Cout;             // Cout % 8 == 0: a 4-channel group is wholly in or out
  float acc[4][4] = {};
  const Gather2 q = gather2_pos<MODE>(src, g, m0 + am);
  float4 ra = conv2_gather<MODE>(q, g, ak);
  float4 rb = bcol && bk < g.K ? *reinterpret_cast<const float4*>(w + (long long)bk * g.Cout + n0 + bn)
                               : make_float4(0.f, 0.f, 0.f, 0.f);
  int buf = 0;
  for (int k0 = 0; k0 < g.K; k0 += FC_BK) {
    As[buf][ak + 0][am] = ra.x; As[buf][ak + 1][am] = ra.y; As[buf][ak + 2][am] = ra.z; As[buf][ak + 3][am] = ra.w;
    *reinterpret_cast<float4*>(&Bs[buf][bk][bn]) = rb;
    __syncthreads();
    const int k1 = k0 + FC_BK;
    if (k1 < g.K) {
      ra = conv2_gather<MODE>(q, g, k1 + ak);
      rb = bcol && k1 + bk < g.K ? *reinterpret_cast<const float4*>(w + (long long)(k1 + bk) * g.Cout + n0 + bn)
                                 : make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll
    for (int kk = 0; kk < FC_BK; ++kk) {
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

const char* conv2d_error(const McvdOp& op) {
  if (!op.src0 || !op.dst || !op.w || !op.bias) return "null input, output, weights or bias";
  if (op.C0 <= 0 || op.C0 % 4) return "input channels must be a positive multiple of 4";
  if (op.Cout <= 0 || op.Cout % 8) return "output channels must be a positive multiple of 8";
  if (op.i0 < 1 || op.i1 < 1 || op.i2 < 1 || op.i3 < 0 || op.i4 < 0) return "kernel, stride or padding out of range";
  if (op.i3 >= op.i0 || op.i4 >= op.i1) return "padding must be smaller than the kernel";
  if (op.i5 < 1) return "input size out of range";
  if (op.flags & ~(MCVD_F_POOL | MCVD_F_AVG)) return "flags other than MCVD_F_POOL and MCVD_F_AVG";
  if ((op.flags & MCVD_F_AVG) && !(op.flags & MCVD_F_POOL)) return "MCVD_F_AVG needs MCVD_F_POOL";
  if ((op.flags & MCVD_F_POOL) && (op.i0 != 1 || op.i1 != 1 || op.i2 != 1 || op.i3 || op.i4))
    return "the fused pool needs a 1x1 stride-1 convolution without padding";
  if (op.i7 < 0 || op.i7 % 4 || op.i6 % 4 || op.i6 < op.i7 + op.Cout)
    return "channel pitch must be a multiple of 4 and at least offset + Cout (offset a multiple of 4)";
  if (op.i5 + 2 * op.i3 < op.i0 || op.i5 + 2 * op.i4 < op.i1) return "kernel larger than the padded input";
  if (op.H != (op.i5 + 2 * op.i3 - op.i0) / op.i2 + 1 || op.W != (op.i5 + 2 * op.i4 - op.i1) / op.i2 + 1)
    return "output size disagrees with the convolution geometry";
  const long long K = (long long)op.i0 * op.i1 * op.C0;
  if (K > (1LL << 30)) return "reduction too long";
  const long long M = (long long)op.B * op.H * op.W;
  if ((M + FC_BM - 1) / FC_BM > 0x7fffffffLL) return "too many output positions for the grid";
  return nullptr;
}

int launch_conv2d(const McvdOp& op, cudaStream_t s) {
  if (const char* why = conv2d_error(op)) MCVD_CHECK(false, "CONV2D: %s", why);
  Conv2Geom g;
  g.Sin = op.i5; g.Cin = op.C0; g.kh = op.i0; g.kw = op.i1; g.stride = op.i2; g.ph = op.i3; g.pw = op.i4;
  g.Ho = op.H; g.Wo = op.W; g.Cout = op.Cout; g.K = op.i0 * op.i1 * op.C0; g.pitch = op.i6; g.off = op.i7;
  g.M = (long long)op.B * op.H * op.W;
  dim3 grid((unsigned)((g.M + FC_BM - 1) / FC_BM), (unsigned)cdiv(op.Cout, FC_BN));
  const float* x = (const float*)op.src0;
  const float* w = (const float*)op.w;
  const float* b = (const float*)op.bias;
  float* y = (float*)op.dst;
  if (op.flags & MCVD_F_POOL) {
    if (op.flags & MCVD_F_AVG) k_conv2d<G_AVGPOOL><<<grid, 256, 0, s>>>(x, w, b, y, g);
    else k_conv2d<G_MAXPOOL><<<grid, 256, 0, s>>>(x, w, b, y, g);
  } else if (op.i0 == 1 && op.i1 == 1 && op.i2 == 1) {
    k_conv2d<G_PW><<<grid, 256, 0, s>>>(x, w, b, y, g);
  } else {
    k_conv2d<G_GENERAL><<<grid, 256, 0, s>>>(x, w, b, y, g);
  }
  MCVD_CUDA_LAUNCH_CHECK("conv2d");
  return 0;
}

// ------------------------------------------------------------------------------------------------
// 3x3 / stride-2 max-pool without padding (nn.MaxPool2d(kernel_size=3, stride=2) and the pool branches of
// InceptionB / InceptionD), into a channel slice.  One thread per output position and 4-channel group.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_maxpool2d(const float4* __restrict__ src, float4* __restrict__ dst, int Sin,
                                                   int C4, int So, int pitch4, int off4, long long total) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int c4 = (int)(idx % C4);
  long long r = idx / C4;
  const int ox = (int)(r % So); r /= So;
  const int oy = (int)(r % So);
  const long long n = r / So;
  const float4* img = src + n * Sin * Sin * C4 + c4;
  float4 v = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
  for (int dy = 0; dy < 3; ++dy)
    for (int dx = 0; dx < 3; ++dx) {
      const float4 u = img[((long long)(2 * oy + dy) * Sin + 2 * ox + dx) * C4];
      v.x = fmaxf(v.x, u.x); v.y = fmaxf(v.y, u.y); v.z = fmaxf(v.z, u.z); v.w = fmaxf(v.w, u.w);
    }
  dst[((n * So + oy) * So + ox) * pitch4 + off4 + c4] = v;
}

const char* maxpool2d_error(const McvdOp& op) {
  if (!op.src0 || !op.dst) return "null input or output";
  if (op.C0 <= 0 || op.C0 % 4) return "channels must be a positive multiple of 4";
  if (op.i5 < 3) return "input smaller than the 3x3 window";
  if (op.H != op.W || op.H != (op.i5 - 3) / 2 + 1) return "output size disagrees with the 3x3 / stride-2 geometry";
  if (op.i7 < 0 || op.i7 % 4 || op.i6 % 4 || op.i6 < op.i7 + op.C0)
    return "channel pitch must be a multiple of 4 and at least offset + C0 (offset a multiple of 4)";
  const long long total = (long long)op.B * op.H * op.W * (op.C0 / 4);
  if ((total + 255) / 256 > 0x7fffffffLL) return "too many outputs for the grid";
  return nullptr;
}

int launch_maxpool2d(const McvdOp& op, cudaStream_t s) {
  if (const char* why = maxpool2d_error(op)) MCVD_CHECK(false, "MAXPOOL2D: %s", why);
  const long long total = (long long)op.B * op.H * op.W * (op.C0 / 4);
  k_maxpool2d<<<(unsigned)((total + 255) / 256), 256, 0, s>>>((const float4*)op.src0, (float4*)op.dst, op.i5,
                                                               op.C0 / 4, op.H, op.i6 / 4, op.i7 / 4, total);
  MCVD_CUDA_LAUNCH_CHECK("maxpool2d");
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
