// LPIPS v0.1 (net-lin, AlexNet backbone) of generated frames against real ones: see MCVD_OP_LPIPS_PREP,
// MCVD_OP_CONV_RELU and MCVD_OP_LPIPS_LAYER in include/mcvd_b200.h.  One chunk of N frame pairs is 11 launches:
// prep, then per AlexNet layer one convolution (conv_eval.cu) and one LPIPS head that consumes its tap.
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
