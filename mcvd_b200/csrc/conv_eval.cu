// fp32 convolutions and max-pools of the evaluation networks: MCVD_OP_CONV_RELU (LPIPS), MCVD_OP_CONV3D and
// MCVD_OP_MAXPOOL3D (I3D), MCVD_OP_CONV2D and MCVD_OP_MAXPOOL2D (Inception-v3) in include/mcvd_b200.h, with the
// geometry and validation of these kinds and of their _TF32 variants (conv_tf32.cu).
#include "conv_eval.cuh"

namespace mcvd {

// ------------------------------------------------------------------------------------------------
// Convolution + bias + ReLU as an fp32 FFMA implicit GEMM over ConvGeom.  64 x 64 output tile per CTA, 16-deep K
// slices, 4 x 4 outputs per thread, the next slice prefetched into registers while the current one is multiplied.
// Cout only needs to be a multiple of 8 (n tiles are masked), and the result goes to channels [off, off + Cout) of a
// pitch-wide output, so an Inception block's branches write their concat in place.  Every output is accumulated by
// one thread in K order, so its value does not depend on the batch or chunk it is computed in.
// ------------------------------------------------------------------------------------------------
constexpr int CE_BM = 64, CE_BN = 64, CE_BK = 16;

template <int MODE, int MIN_BLOCKS>
__global__ void __launch_bounds__(256, MIN_BLOCKS)
    k_conv_ffma(const float* __restrict__ src, const float* __restrict__ w, const float* __restrict__ bias,
                float* __restrict__ dst, ConvGeom g) {
  __shared__ __align__(16) float As[2][CE_BK][CE_BM];
  __shared__ __align__(16) float Bs[2][CE_BK][CE_BN];
  const int tid = threadIdx.x;
  const long long m0 = (long long)blockIdx.x * CE_BM;
  const int n0 = blockIdx.y * CE_BN;
  // loader roles: A = one position x 4 consecutive k (4 channels of one tap); B = one k row x 4 output channels
  const int am = tid % CE_BM, ak = (tid / CE_BM) * 4;
  const int bk = tid / (CE_BN / 4), bn = (tid % (CE_BN / 4)) * 4;
  const int tm = (tid / 16) * 4, tn = (tid % 16) * 4;
  const bool bcol = n0 + bn < g.Cout;             // Cout % 8 == 0: a 4-channel group is wholly in or out
  float acc[4][4] = {};
  const ConvPos q = conv_pos<MODE>(src, g, m0 + am);
  // a position past M or a k past K reads zero; checked before k is decomposed, which keeps the loop's integer work
  // to the taps that are read
  const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
  float4 ra = q.img && ak < g.K ? conv_gather<MODE, false>(q, g, conv_tap<MODE>(g, ak)) : zero;
  float4 rb = bcol && bk < g.K ? ld4(w + (long long)bk * g.Cout + n0 + bn) : zero;
  int buf = 0;
  for (int k0 = 0; k0 < g.K; k0 += CE_BK) {
    As[buf][ak + 0][am] = ra.x; As[buf][ak + 1][am] = ra.y; As[buf][ak + 2][am] = ra.z; As[buf][ak + 3][am] = ra.w;
    *reinterpret_cast<float4*>(&Bs[buf][bk][bn]) = rb;
    __syncthreads();
    const int k1 = k0 + CE_BK;
    if (k1 < g.K) {
      ra = q.img && k1 + ak < g.K ? conv_gather<MODE, false>(q, g, conv_tap<MODE>(g, k1 + ak)) : zero;
      rb = bcol && k1 + bk < g.K ? ld4(w + (long long)(k1 + bk) * g.Cout + n0 + bn) : zero;
    }
#pragma unroll
    for (int kk = 0; kk < CE_BK; ++kk) {
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
  const float4 bb = ld4(bias + n0 + tn);
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

template <int MODE, int MIN_BLOCKS>
static void run_conv_ffma(const McvdOp& op, const ConvGeom& g, cudaStream_t s) {
  dim3 grid((unsigned)((g.M + CE_BM - 1) / CE_BM), (unsigned)cdiv(g.Cout, CE_BN));
  k_conv_ffma<MODE, MIN_BLOCKS><<<grid, 256, 0, s>>>((const float*)op.src0, (const float*)op.w,
                                                     (const float*)op.bias, (float*)op.dst, g);
}

int launch_conv_ffma(const McvdOp& op, cudaStream_t s) {
  const char* name = conv_kind_name(op.kind);
  MCVD_CHECK(op.src0 && op.dst, "%s: null pointer", name);
  ConvGeom g;
  if (const char* why = conv_geom(op, g)) MCVD_CHECK(false, "%s: %s", name, why);
  const int mode = gather_mode(op);
  if (op.kind == MCVD_OP_CONV_RELU) {              // the AlexNet layers leave occupancy to the compiler (0)
    if (mode == G_S2MAX) run_conv_ffma<G_S2MAX, 0>(op, g, s);
    else run_conv_ffma<G_CONV2, 0>(op, g, s);
  } else {                                         // the branch pools need more registers than 4 CTAs per SM leave
    switch (mode) {
      case G_CONV2: run_conv_ffma<G_CONV2, 4>(op, g, s); break;
      case G_CONV3: run_conv_ffma<G_CONV3, 4>(op, g, s); break;
      case G_PW: run_conv_ffma<G_PW, 4>(op, g, s); break;
      case G_BMAX: run_conv_ffma<G_BMAX, 2>(op, g, s); break;
      default: run_conv_ffma<G_BAVG, 2>(op, g, s); break;
    }
  }
  MCVD_CUDA_LAUNCH_CHECK(name);
  return 0;
}

// ------------------------------------------------------------------------------------------------
// Max-pool over ConvGeom (window kt x kh x kw, strides, front pads) into a channel slice.  Out-of-map taps read zero
// and take part in the max, as in I3D's MaxPool3dSamePadding.  MAXPOOL2D (!T3) is 3x3 / stride 2 without padding by
// definition: its window is unrolled and never leaves the map.  One thread per output position and 4-channel group.
// ------------------------------------------------------------------------------------------------
template <bool T3>
__global__ void __launch_bounds__(256) k_maxpool(const float4* __restrict__ src, float4* __restrict__ dst, ConvGeom g,
                                                 long long total) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int C4 = g.Cin >> 2;
  const int c4 = (int)(idx % C4);
  const long long p = idx / C4;                    // output position
  long long r = p;
  const int ox = (int)(r % g.Wo); r /= g.Wo;
  const int oy = (int)(r % g.Ho); r /= g.Ho;
  int ot = 0;
  if (T3) {
    ot = (int)(r % g.To);
    r /= g.To;
  }
  const float4* img = src + r * (T3 ? g.Tin : 1) * g.Hin * g.Win * C4 + c4;
  const int t0 = ot * g.st - g.pt, y0 = oy * g.ss - g.ph, x0 = ox * g.ss - g.pw;
  const int kt = T3 ? g.kt : 1, kh = T3 ? g.kh : 3, kw = T3 ? g.kw : 3;
  float4 v = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
  for (int dt = 0; dt < kt; ++dt)
    for (int dy = 0; dy < kh; ++dy)
      for (int dx = 0; dx < kw; ++dx) {
        const int it = t0 + dt, iy = y0 + dy, ix = x0 + dx;
        float4 u = make_float4(0.f, 0.f, 0.f, 0.f);
        if (!T3 || (it >= 0 && it < g.Tin && iy >= 0 && iy < g.Hin && ix >= 0 && ix < g.Win))
          u = img[(((long long)it * g.Hin + iy) * g.Win + ix) * C4];
        max4(v, u);
      }
  dst[p * (g.pitch >> 2) + (g.off >> 2) + c4] = v;
}

int launch_maxpool(const McvdOp& op, cudaStream_t s) {
  const char* name = conv_kind_name(op.kind);
  ConvGeom g;
  if (const char* why = conv_geom(op, g)) MCVD_CHECK(false, "%s: %s", name, why);
  const long long total = g.M * (g.Cin / 4);
  const unsigned blocks = (unsigned)((total + 255) / 256);
  if (op.kind == MCVD_OP_MAXPOOL3D) k_maxpool<true><<<blocks, 256, 0, s>>>((const float4*)op.src0, (float4*)op.dst,
                                                                           g, total);
  else k_maxpool<false><<<blocks, 256, 0, s>>>((const float4*)op.src0, (float4*)op.dst, g, total);
  MCVD_CUDA_LAUNCH_CHECK(name);
  return 0;
}

// ------------------------------------------------------------------------------------------------
// geometry and validation
// ------------------------------------------------------------------------------------------------
// channels [i7, i7 + width) do not fit a pitch-wide output, or pitch or offset is not a multiple of 4
static bool bad_slice(const McvdOp& op, int width) {
  return op.i7 < 0 || op.i7 % 4 || op.i6 % 4 || op.i6 < op.i7 + width;
}

static bool grid_too_big(long long units, int per_cta) { return (units + per_cta - 1) / per_cta > 0x7fffffffLL; }

static void set_2d(ConvGeom& g, int Hin, int Win, int kh, int kw, int stride, int ph, int pw, int Ho, int Wo) {
  g.Tin = 1; g.Hin = g.Hc = Hin; g.Win = g.Wc = Win;
  g.kt = 1; g.kh = kh; g.kw = kw; g.st = 1; g.ss = stride; g.pt = 0; g.ph = ph; g.pw = pw;
  g.To = 1; g.Ho = Ho; g.Wo = Wo;
}

// I3D's TF-SAME geometry: time i4, side i5, window i0 x i1 x i1, stride i2 x i3 x i3
static void set_same_3d(ConvGeom& g, const McvdOp& op) {
  g.Tin = op.i4; g.Hin = g.Win = g.Hc = g.Wc = op.i5;
  g.kt = op.i0; g.kh = g.kw = op.i1; g.st = op.i2; g.ss = op.i3;
  g.pt = same_pad(op.i4, op.i0, op.i2) / 2;
  g.ph = g.pw = same_pad(op.i5, op.i1, op.i3) / 2;
  g.To = same_out(op.i4, op.i0, op.i2); g.Ho = g.Wo = op.H;
}

static const char* conv_relu_geom(const McvdOp& op, ConvGeom& g) {
  if (!op.w || !op.bias) return "null weights or bias";
  if (op.C0 <= 0 || op.C0 % 4) return "input channels must be a positive multiple of 4";
  if (op.Cout <= 0 || op.Cout % CE_BN) return "output channels must be a positive multiple of 64";
  if (op.i0 < 1 || op.i1 < 1 || op.i2 < 0) return "kernel size, stride or padding out of range";
  if (op.i3 < 1 || op.i4 < 1) return "input size out of range";
  const bool pool = (op.flags & MCVD_F_POOL) != 0;
  if (pool && (op.i3 < 3 || op.i4 < 3)) return "pooled input smaller than the 3x3 window";
  const int hc = pool ? (op.i3 - 3) / 2 + 1 : op.i3, wc = pool ? (op.i4 - 3) / 2 + 1 : op.i4;
  if (hc + 2 * op.i2 < op.i0 || wc + 2 * op.i2 < op.i0) return "kernel larger than the padded input";
  if (op.H != (hc + 2 * op.i2 - op.i0) / op.i1 + 1 || op.W != (wc + 2 * op.i2 - op.i0) / op.i1 + 1)
    return "output size disagrees with the convolution geometry";
  set_2d(g, op.i3, op.i4, op.i0, op.i0, op.i1, op.i2, op.i2, op.H, op.W);
  g.Hc = hc; g.Wc = wc;
  g.Cin = op.C0; g.Cout = g.pitch = op.Cout; g.off = 0;
  g.K = op.i0 * op.i0 * op.C0;
  g.M = (long long)op.B * op.H * op.W;
  return nullptr;
}

static const char* conv3d_geom(const McvdOp& op, ConvGeom& g) {
  if (!op.src0 || !op.dst || !op.w || !op.bias) return "null input, output, weights or bias";
  if (op.C0 <= 0 || op.C0 % 4) return "input channels must be a positive multiple of 4";
  if (op.Cout <= 0 || op.Cout % 8) return "output channels must be a positive multiple of 8";
  if (op.i0 < 1 || op.i1 < 1 || op.i2 < 1 || op.i3 < 1) return "kernel size or stride out of range";
  if (op.i4 < 1 || op.i5 < 1) return "input size out of range";
  if (bad_slice(op, op.Cout))
    return "channel pitch must be a multiple of 4 and at least offset + Cout (offset a multiple of 4)";
  if (op.H != op.W || op.H != same_out(op.i5, op.i1, op.i3)) return "output size disagrees with the SAME geometry";
  const long long K = (long long)op.i0 * op.i1 * op.i1 * op.C0;
  if (K > (1LL << 30)) return "reduction too long";
  set_same_3d(g, op);
  g.Cin = op.C0; g.Cout = op.Cout; g.pitch = op.i6; g.off = op.i7;
  g.K = (int)K;
  g.M = (long long)op.B * g.To * op.H * op.W;
  return grid_too_big(g.M, CE_BM) ? "too many output positions for the grid" : nullptr;
}

static const char* maxpool3d_geom(const McvdOp& op, ConvGeom& g) {
  if (!op.src0 || !op.dst) return "null input or output";
  if (op.C0 <= 0 || op.C0 % 4) return "channels must be a positive multiple of 4";
  if (op.i0 < 1 || op.i1 < 1 || op.i2 < 1 || op.i3 < 1) return "window or stride out of range";
  if (op.i4 < 1 || op.i5 < 1) return "input size out of range";
  if (op.H != op.W || op.H != same_out(op.i5, op.i1, op.i3)) return "output size disagrees with the SAME geometry";
  set_same_3d(g, op);
  g.Cin = g.Cout = g.pitch = op.C0; g.off = 0; g.K = 0;
  g.M = (long long)op.B * g.To * op.H * op.W;
  return grid_too_big(g.M * (op.C0 / 4), 256) ? "too many outputs for the grid" : nullptr;
}

static const char* conv2d_geom(const McvdOp& op, ConvGeom& g) {
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
  if (bad_slice(op, op.Cout))
    return "channel pitch must be a multiple of 4 and at least offset + Cout (offset a multiple of 4)";
  if (op.i5 + 2 * op.i3 < op.i0 || op.i5 + 2 * op.i4 < op.i1) return "kernel larger than the padded input";
  if (op.H != (op.i5 + 2 * op.i3 - op.i0) / op.i2 + 1 || op.W != (op.i5 + 2 * op.i4 - op.i1) / op.i2 + 1)
    return "output size disagrees with the convolution geometry";
  const long long K = (long long)op.i0 * op.i1 * op.C0;
  if (K > (1LL << 30)) return "reduction too long";
  set_2d(g, op.i5, op.i5, op.i0, op.i1, op.i2, op.i3, op.i4, op.H, op.W);
  g.Cin = op.C0; g.Cout = op.Cout; g.pitch = op.i6; g.off = op.i7;
  g.K = (int)K;
  g.M = (long long)op.B * op.H * op.W;
  return grid_too_big(g.M, CE_BM) ? "too many output positions for the grid" : nullptr;
}

static const char* maxpool2d_geom(const McvdOp& op, ConvGeom& g) {
  if (!op.src0 || !op.dst) return "null input or output";
  if (op.C0 <= 0 || op.C0 % 4) return "channels must be a positive multiple of 4";
  if (op.i5 < 3) return "input smaller than the 3x3 window";
  if (op.H != op.W || op.H != (op.i5 - 3) / 2 + 1) return "output size disagrees with the 3x3 / stride-2 geometry";
  if (bad_slice(op, op.C0))
    return "channel pitch must be a multiple of 4 and at least offset + C0 (offset a multiple of 4)";
  set_2d(g, op.i5, op.i5, 3, 3, 2, 0, 0, op.H, op.W);
  g.Cin = g.Cout = op.C0; g.pitch = op.i6; g.off = op.i7; g.K = 0;
  g.M = (long long)op.B * op.H * op.W;
  return grid_too_big(g.M * (op.C0 / 4), 256) ? "too many outputs for the grid" : nullptr;
}

const char* conv_geom(const McvdOp& op, ConvGeom& g) {
  switch (op.kind) {
    case MCVD_OP_CONV_RELU:
    case MCVD_OP_CONV_RELU_TF32: return conv_relu_geom(op, g);
    case MCVD_OP_CONV3D:
    case MCVD_OP_CONV3D_TF32: return conv3d_geom(op, g);
    case MCVD_OP_MAXPOOL3D: return maxpool3d_geom(op, g);
    case MCVD_OP_CONV2D:
    case MCVD_OP_CONV2D_TF32: return conv2d_geom(op, g);
    case MCVD_OP_MAXPOOL2D: return maxpool2d_geom(op, g);
    default: return "not a convolution or max-pool kind";
  }
}

int gather_mode(const McvdOp& op) {
  switch (op.kind) {
    case MCVD_OP_CONV_RELU:
    case MCVD_OP_CONV_RELU_TF32: return (op.flags & MCVD_F_POOL) ? G_S2MAX : G_CONV2;
    case MCVD_OP_CONV3D:
    case MCVD_OP_CONV3D_TF32: return op.i0 == 1 && op.i1 == 1 && op.i2 == 1 && op.i3 == 1 ? G_PW : G_CONV3;
    default:
      if (op.flags & MCVD_F_POOL) return (op.flags & MCVD_F_AVG) ? G_BAVG : G_BMAX;
      return op.i0 == 1 && op.i1 == 1 && op.i2 == 1 ? G_PW : G_CONV2;
  }
}

const char* conv_kind_name(int kind) {
  switch (kind) {
    case MCVD_OP_CONV_RELU: return "CONV_RELU";
    case MCVD_OP_CONV3D: return "CONV3D";
    case MCVD_OP_MAXPOOL3D: return "MAXPOOL3D";
    case MCVD_OP_CONV2D: return "CONV2D";
    case MCVD_OP_MAXPOOL2D: return "MAXPOOL2D";
    case MCVD_OP_CONV3D_TF32: return "CONV3D_TF32";
    case MCVD_OP_CONV2D_TF32: return "CONV2D_TF32";
    case MCVD_OP_CONV_RELU_TF32: return "CONV_RELU_TF32";
    default: return "?";
  }
}

}  // namespace mcvd
