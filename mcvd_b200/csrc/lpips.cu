// LPIPS v0.1 (net-lin, AlexNet backbone) of generated frames against real ones: see MCVD_OP_LPIPS_PREP,
// MCVD_OP_CONV_RELU and MCVD_OP_LPIPS_LAYER in include/mcvd_b200.h.  One chunk of N frame pairs is 11 launches:
// prep, then per AlexNet layer one convolution and one LPIPS head that consumes its tap.
#include "mcvd_common.cuh"

namespace mcvd {

// ------------------------------------------------------------------------------------------------
// prep: clamp, ToPILImage (trunc(x*255)), PIL bilinear resize to 128x128 in Pillow's 8-bit fixed point
// (horizontal pass, then vertical pass, each rounded and clipped to uint8), ToTensor, Normalize(0.5, 0.5),
// ScalingLayer -- all fp32 in torchvision's order, so the network input is bit-identical to the reference's.
// One thread per output pixel of one image; images [0, N) are pred frames, [N, 2N) real frames.
// ------------------------------------------------------------------------------------------------
constexpr int LP_SIDE = 128;
constexpr int LP_PREC = 22;                        // Pillow's PRECISION_BITS for 8-bit images

__device__ __forceinline__ int pil_clip8(int v) {
  if (v >= (1 << LP_PREC << 8)) return 255;
  if (v <= 0) return 0;
  return v >> LP_PREC;
}

__device__ __forceinline__ int frame_u8(const float* p) {
  const float x = fminf(fmaxf(*p, 0.0f), 1.0f);
  return (int)(x * 255.0f);                        // ToPILImage: mul(255).byte()
}

__global__ void __launch_bounds__(256) k_lpips_prep(const float* __restrict__ pred, const float* __restrict__ real,
                                                    const int* __restrict__ table, float* __restrict__ dst, int N,
                                                    int C, int nf, int S, int K) {
  const int pix = blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= LP_SIDE * LP_SIDE) return;
  const int img = blockIdx.y;                      // 0 .. 2N-1
  const int oy = pix / LP_SIDE, ox = pix % LP_SIDE;
  const int pair = img < N ? img : img - N;        // frame index over (clip, frame)
  const int b = pair / nf, f = pair % nf;
  const float* base = (img < N ? pred : real) + ((long long)b * nf + f) * C * S * S;
  const int* ty = table + oy * (2 + K);
  const int* tx = table + ox * (2 + K);
  const int y0 = ty[0], ny = ty[1], x0 = tx[0], nx = tx[1];
  int out[3];
  for (int c = 0; c < C; ++c) {
    const float* plane = base + (long long)c * S * S;
    int acc = 1 << (LP_PREC - 1);
    for (int j = 0; j < ny; ++j) {
      const float* row = plane + (long long)(y0 + j) * S + x0;
      int h = 1 << (LP_PREC - 1);
      for (int i = 0; i < nx; ++i) h += frame_u8(row + i) * tx[2 + i];
      acc += pil_clip8(h) * ty[2 + j];
    }
    out[c] = pil_clip8(acc);
  }
  const float shift[3] = {-.030f, -.088f, -.188f}, scale[3] = {.458f, .448f, .450f};
  float4 v;
  float* pv = &v.x;
  for (int c = 0; c < 3; ++c) {
    float t = (float)out[C == 1 ? 0 : c] / 255.0f;  // ToTensor
    t = (t - 0.5f) / 0.5f;                           // Normalize(0.5, 0.5)
    pv[c] = (t - shift[c]) / scale[c];               // ScalingLayer
  }
  v.w = 0.0f;
  reinterpret_cast<float4*>(dst)[(long long)img * LP_SIDE * LP_SIDE + pix] = v;
}

int launch_lpips_prep(const McvdOp& op, cudaStream_t s) {
  MCVD_CHECK(op.src0 && op.src1 && op.w && op.dst, "LPIPS_PREP: null pointer");
  MCVD_CHECK(op.C0 == 1 || op.C0 == 3, "LPIPS_PREP: %d channels per frame (1 or 3)", op.C0);
  MCVD_CHECK(op.H == LP_SIDE && op.W == LP_SIDE, "LPIPS_PREP: output side %dx%d (must be 128x128)", op.H, op.W);
  MCVD_CHECK(op.i0 >= 1 && op.i1 >= 1 && op.i2 >= 1, "LPIPS_PREP: frames %d, input side %d, taps %d", op.i0, op.i1,
             op.i2);
  const long long images = 2LL * op.B * op.i0;
  MCVD_CHECK(images <= 65535, "LPIPS_PREP: %lld images too many for the grid", images);
  dim3 grid(LP_SIDE * LP_SIDE / 256, (unsigned)images);
  k_lpips_prep<<<grid, 256, 0, s>>>((const float*)op.src0, (const float*)op.src1, (const int*)op.w, (float*)op.dst,
                                    op.B * op.i0, op.C0, op.i0, op.i1, op.i2);
  MCVD_CUDA_LAUNCH_CHECK("lpips_prep");
  return 0;
}

// ------------------------------------------------------------------------------------------------
// NHWC direct convolution + bias + ReLU as an fp32 FFMA implicit GEMM: M = images * OH * OW output positions,
// N = Cout, K = k * k * Cin in (ky, kx, c) order.  64 x 64 output tile per CTA, 16-deep K slices, 4 x 4 outputs
// per thread, the next slice prefetched into registers while the current one is multiplied.  Every output is
// accumulated by one thread in K order, so its value does not depend on the batch it is computed in.
// POOL: the conv reads the 3x3/s2 max-pool of src (AlexNet features[2], [5]) instead of src itself.
// ------------------------------------------------------------------------------------------------
constexpr int CR_BM = 64, CR_BN = 64, CR_BK = 16;

struct ConvGeom {
  int Hin, Win, Hc, Wc, Cin, ks, stride, pad, OH, OW, Cout, K;
  long long M;
};

// the output position one A-loader thread gathers for, decomposed once per CTA (not once per K slice)
struct GatherPos {
  const float* img;          // the position's image, NULL past the last position
  int iy0, ix0;              // top-left input coordinate of its window
};

__device__ __forceinline__ GatherPos gather_pos(const float* __restrict__ src, const ConvGeom& g, long long m) {
  GatherPos q{nullptr, 0, 0};
  if (m >= g.M) return q;
  const int P = g.OH * g.OW;
  const long long n = m / P;
  const int r = (int)(m - n * P);
  q.img = src + n * g.Hin * g.Win * g.Cin;
  q.iy0 = (r / g.OW) * g.stride - g.pad;
  q.ix0 = (r % g.OW) * g.stride - g.pad;
  return q;
}

template <bool POOL>
__device__ __forceinline__ float4 conv_gather(const GatherPos& q, const ConvGeom& g, int k) {
  const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
  if (!q.img || k >= g.K) return zero;
  const int tap = k / g.Cin, c = k - tap * g.Cin;
  const int ky = tap / g.ks;
  const int iy = q.iy0 + ky, ix = q.ix0 + tap - ky * g.ks;
  if (iy < 0 || iy >= g.Hc || ix < 0 || ix >= g.Wc) return zero;
  const float* img = q.img + c;
  if (!POOL) return *reinterpret_cast<const float4*>(img + ((long long)iy * g.Win + ix) * g.Cin);
  float4 v = *reinterpret_cast<const float4*>(img + ((long long)(2 * iy) * g.Win + 2 * ix) * g.Cin);
#pragma unroll
  for (int dy = 0; dy < 3; ++dy)
#pragma unroll
    for (int dx = 0; dx < 3; ++dx) {
      if (dy == 0 && dx == 0) continue;
      const float4 u = *reinterpret_cast<const float4*>(img + ((long long)(2 * iy + dy) * g.Win + 2 * ix + dx) * g.Cin);
      v.x = fmaxf(v.x, u.x); v.y = fmaxf(v.y, u.y); v.z = fmaxf(v.z, u.z); v.w = fmaxf(v.w, u.w);
    }
  return v;
}

template <bool POOL>
__global__ void __launch_bounds__(256) k_conv_relu(const float* __restrict__ src, const float* __restrict__ w,
                                                   const float* __restrict__ bias, float* __restrict__ dst, ConvGeom g) {
  __shared__ __align__(16) float As[2][CR_BK][CR_BM];
  __shared__ __align__(16) float Bs[2][CR_BK][CR_BN];
  const int tid = threadIdx.x;
  const long long m0 = (long long)blockIdx.x * CR_BM;
  const int n0 = blockIdx.y * CR_BN;
  // loader roles: A = one position x 4 consecutive k (4 channels of one tap); B = one k row x 4 output channels
  const int am = tid % CR_BM, ak = (tid / CR_BM) * 4;
  const int bk = tid / (CR_BN / 4), bn = (tid % (CR_BN / 4)) * 4;
  const int tm = (tid / 16) * 4, tn = (tid % 16) * 4;
  float acc[4][4] = {};
  const GatherPos q = gather_pos(src, g, m0 + am);
  float4 ra = conv_gather<POOL>(q, g, ak);
  float4 rb = bk < g.K ? *reinterpret_cast<const float4*>(w + (long long)bk * g.Cout + n0 + bn)
                       : make_float4(0.f, 0.f, 0.f, 0.f);
  int buf = 0;
  for (int k0 = 0; k0 < g.K; k0 += CR_BK) {
    As[buf][ak + 0][am] = ra.x; As[buf][ak + 1][am] = ra.y; As[buf][ak + 2][am] = ra.z; As[buf][ak + 3][am] = ra.w;
    *reinterpret_cast<float4*>(&Bs[buf][bk][bn]) = rb;
    __syncthreads();
    const int k1 = k0 + CR_BK;
    if (k1 < g.K) {
      ra = conv_gather<POOL>(q, g, k1 + ak);
      rb = k1 + bk < g.K ? *reinterpret_cast<const float4*>(w + (long long)(k1 + bk) * g.Cout + n0 + bn)
                         : make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll
    for (int kk = 0; kk < CR_BK; ++kk) {
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
    *reinterpret_cast<float4*>(dst + m * g.Cout + n0 + tn) = o;
  }
}

// NULL, or why the geometry of a MCVD_OP_CONV_RELU op is unusable (shared by validation and launch)
const char* conv_relu_error(const McvdOp& op) {
  if (!op.w || !op.bias) return "null weights or bias";
  if (op.C0 <= 0 || op.C0 % 4) return "input channels must be a positive multiple of 4";
  if (op.Cout <= 0 || op.Cout % CR_BN) return "output channels must be a positive multiple of 64";
  if (op.i0 < 1 || op.i1 < 1 || op.i2 < 0) return "kernel size, stride or padding out of range";
  if (op.i3 < 1 || op.i4 < 1) return "input size out of range";
  const bool pool = (op.flags & MCVD_F_POOL) != 0;
  if (pool && (op.i3 < 3 || op.i4 < 3)) return "pooled input smaller than the 3x3 window";
  const int hc = pool ? (op.i3 - 3) / 2 + 1 : op.i3, wc = pool ? (op.i4 - 3) / 2 + 1 : op.i4;
  if (hc + 2 * op.i2 < op.i0 || wc + 2 * op.i2 < op.i0) return "kernel larger than the padded input";
  if (op.H != (hc + 2 * op.i2 - op.i0) / op.i1 + 1 || op.W != (wc + 2 * op.i2 - op.i0) / op.i1 + 1)
    return "output size disagrees with the convolution geometry";
  return nullptr;
}

int launch_conv_relu(const McvdOp& op, cudaStream_t s) {
  MCVD_CHECK(op.src0 && op.dst, "CONV_RELU: null pointer");
  if (const char* why = conv_relu_error(op)) MCVD_CHECK(false, "CONV_RELU: %s", why);
  const bool pool = (op.flags & MCVD_F_POOL) != 0;
  ConvGeom g;
  g.Hin = op.i3; g.Win = op.i4; g.Cin = op.C0; g.ks = op.i0; g.stride = op.i1; g.pad = op.i2;
  g.Hc = pool ? (op.i3 - 3) / 2 + 1 : op.i3;
  g.Wc = pool ? (op.i4 - 3) / 2 + 1 : op.i4;
  g.OH = op.H; g.OW = op.W; g.Cout = op.Cout; g.K = op.i0 * op.i0 * op.C0;
  g.M = (long long)op.B * op.H * op.W;
  dim3 grid((unsigned)((g.M + CR_BM - 1) / CR_BM), op.Cout / CR_BN);
  if (pool) k_conv_relu<true><<<grid, 256, 0, s>>>((const float*)op.src0, (const float*)op.w, (const float*)op.bias,
                                                   (float*)op.dst, g);
  else k_conv_relu<false><<<grid, 256, 0, s>>>((const float*)op.src0, (const float*)op.w, (const float*)op.bias,
                                               (float*)op.dst, g);
  MCVD_CUDA_LAUNCH_CHECK("conv_relu");
  return 0;
}

// ------------------------------------------------------------------------------------------------
// LPIPS head of one tap: per position, unit-normalise both feature vectors over channels (f / (|f| + 1e-10)),
// weight the squared difference with lin_k, sum over channels; mean over positions.  One CTA per frame pair,
// one warp per position, fp64 throughout, fixed reduction order, no atomics.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_lpips_layer(const float* __restrict__ f0, const float* __restrict__ f1,
                                                     const float* __restrict__ lin, double* __restrict__ out, int P,
                                                     int C, int accumulate) {
  __shared__ double red[8];
  const int pair = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const float* a = f0 + (long long)pair * P * C;
  const float* b = f1 + (long long)pair * P * C;
  double total = 0.0;
  for (int p = warp; p < P; p += 8) {
    const float* pa = a + (long long)p * C;
    const float* pb = b + (long long)p * C;
    double sa = 0.0, sb = 0.0;
    for (int c = lane; c < C; c += 32) {
      const double x = pa[c], y = pb[c];
      sa += x * x;
      sb += y * y;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      sa += __shfl_xor_sync(0xffffffffu, sa, o);
      sb += __shfl_xor_sync(0xffffffffu, sb, o);
    }
    const double ia = 1.0 / (sqrt(sa) + 1e-10), ib = 1.0 / (sqrt(sb) + 1e-10);
    double d = 0.0;
    for (int c = lane; c < C; c += 32) {
      const double e = __dmul_rn(pa[c], ia) - __dmul_rn(pb[c], ib);   // no FMA: d(a, b) == d(b, a) bit for bit
      d += (double)lin[c] * e * e;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) d += __shfl_xor_sync(0xffffffffu, d, o);
    total += d;
  }
  if (lane == 0) red[warp] = total;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int i = 0; i < 8; ++i) t += red[i];
    t /= (double)P;
    out[pair] = accumulate ? out[pair] + t : t;
  }
}

int launch_lpips_layer(const McvdOp& op, cudaStream_t s) {
  MCVD_CHECK(op.src0 && op.src1 && op.w && op.dst, "LPIPS_LAYER: null pointer");
  MCVD_CHECK(op.C0 >= 1, "LPIPS_LAYER: %d channels", op.C0);
  k_lpips_layer<<<op.B, 256, 0, s>>>((const float*)op.src0, (const float*)op.src1, (const float*)op.w,
                                     (double*)op.dst, op.H * op.W, op.C0, op.i0 != 0);
  MCVD_CUDA_LAUNCH_CHECK("lpips_layer");
  return 0;
}

}  // namespace mcvd
