// Denoising score-matching test loss around the lowered network (see MCVD_OP_DSM_PERTURB / MCVD_OP_DSM_LOSS in
// include/mcvd_b200.h; reference losses/dsm.py:anneal_dsm_score_estimation):
//   perturb:  z keyed by (seed, clip, step tag, element) or injected, x_t = sqrt(a_b) x + sqrt(1 - a_b) z;
//   loss:     per clip, sum of 0.5 (z - eps)^2 or |z - eps| in fp64, one CTA per clip, fixed reduction order.
#include <cmath>

#include "mcvd_common.cuh"
#include "philox.cuh"

namespace mcvd {

// tab[b] = (sqrt(a_b), sqrt(1 - a_b), Gamma shape k_b, Gamma scale s_b).  x_t is two rounded fp32 products and one
// rounded add, as torch evaluates the reference's expression, so with injected z the result is the same bits.
// Grid: x = pixel blocks of one (clip, channel) plane, y = planes (strided when there are more than 65535), so the
// indices need no 64-bit division.
template <bool GAMMA>
__global__ void __launch_bounds__(256) k_dsm_perturb(const float* __restrict__ x, const float4* __restrict__ tab,
                                                     const float* __restrict__ zin, float* __restrict__ xt,
                                                     float* __restrict__ zout, int planes, int C, int HW, int philox,
                                                     uint32_t seed_lo, uint32_t seed_hi, int clip0, int step) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= HW) return;
  for (int plane = blockIdx.y; plane < planes; plane += gridDim.y) {
    const int b = plane / C, c = plane - b * C;
    const long long i = (long long)plane * HW + p;
    const float4 t = tab[b];
    float zv;
    if (GAMMA)
      zv = (float)((double)t.w * philox_gamma_centred((double)t.z, seed_lo, seed_hi, (uint32_t)(clip0 + b),
                                                      (uint32_t)step, (uint32_t)(c * HW + p)));
    else if (philox) zv = philox_normal(seed_lo, seed_hi, (uint32_t)(clip0 + b), (uint32_t)step, (uint32_t)(c * HW + p));
    else zv = zin[i];
    xt[i] = __fadd_rn(__fmul_rn(t.x, x[i]), __fmul_rn(t.y, zv));
    if (zout) zout[i] = zv;
  }
}

// One CTA of DSM_LOSS_THREADS threads per clip: thread j takes the pixels j, j + DSM_LOSS_THREADS, ... and every
// channel of each (eps rows are contiguous in NHWC), accumulating in fp64; the CTA then reduces its partials in a fixed
// tree.  A clip's sum therefore depends only on its own elements, never on the batch size or its position in the
// batch.  1024 threads keep enough loads in flight with only B CTAs on the GPU.
#define DSM_LOSS_THREADS 1024

__global__ void __launch_bounds__(DSM_LOSS_THREADS) k_dsm_loss(const float* __restrict__ eps,
                                                               const float* __restrict__ z, double* __restrict__ out,
                                                               int C, int HW, int pitch, int l1) {
  const int b = blockIdx.x;
  const float* zb = z + (long long)b * C * HW;
  const float* eb = eps + (long long)b * HW * pitch;
  double acc = 0.0;
#pragma unroll 4
  for (int p = threadIdx.x; p < HW; p += DSM_LOSS_THREADS) {
    const float* e = eb + (long long)p * pitch;
    for (int c = 0; c < C; ++c) {
      const float d = __fsub_rn(zb[(long long)c * HW + p], e[c]);      // the reference's fp32 difference
      acc += l1 ? fabs((double)d) : 0.5 * (double)d * (double)d;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_down_sync(0xffffffffu, acc, o);
  __shared__ double warp_sum[DSM_LOSS_THREADS / 32];
  if ((threadIdx.x & 31) == 0) warp_sum[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x < 32) {
    double s = warp_sum[threadIdx.x];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_down_sync(0xffffffffu, s, o);
    if (threadIdx.x == 0) out[b] = s;
  }
}

const char* dsm_error(const McvdOp& op) {
  if (!op.src0 || !op.dst) return "null src0/dst";
  if (op.C0 < 1) return "no channels";
  if (op.kind == MCVD_OP_DSM_PERTURB) {
    if (op.flags & ~(MCVD_F_PHILOX | MCVD_F_GAMMA)) return "flags other than MCVD_F_PHILOX | MCVD_F_GAMMA";
    if ((op.flags & MCVD_F_GAMMA) && !(op.flags & MCVD_F_PHILOX)) return "MCVD_F_GAMMA needs MCVD_F_PHILOX";
    if (!op.aux0) return "null coefficient table aux0";
    if ((op.flags & MCVD_F_PHILOX) && !op.dst2) return "null noise output dst2";
    if (!(op.flags & MCVD_F_PHILOX) && !op.src1) return "null injected noise src1";
    return nullptr;
  }
  if (op.flags & ~MCVD_F_L1) return "flags other than MCVD_F_L1";
  if (!op.src1) return "null noise src1";
  if (op.Cout != 0 && op.Cout < op.C0) return "eps channel pitch Cout below C0";
  return nullptr;
}

int launch_dsm_perturb(const McvdOp& op, cudaStream_t s) {
  const char* why = dsm_error(op);
  MCVD_CHECK(!why, "DSM_PERTURB: %s", why);
  const int planes = op.B * op.C0, HW = op.H * op.W;
  auto kern = (op.flags & MCVD_F_GAMMA) ? k_dsm_perturb<true> : k_dsm_perturb<false>;
  kern<<<dim3((unsigned)cdiv(HW, 256), (unsigned)(planes < 65535 ? planes : 65535)), 256, 0, s>>>(
      (const float*)op.src0, (const float4*)op.aux0, (const float*)op.src1, (float*)op.dst, (float*)op.dst2, planes,
      op.C0, HW, (op.flags & MCVD_F_PHILOX) ? 1 : 0, (uint32_t)op.i0, (uint32_t)op.i1, op.i2, op.i3);
  MCVD_CUDA_LAUNCH_CHECK("dsm_perturb");
  return 0;
}

int launch_dsm_loss(const McvdOp& op, cudaStream_t s) {
  const char* why = dsm_error(op);
  MCVD_CHECK(!why, "DSM_LOSS: %s", why);
  k_dsm_loss<<<(unsigned)op.B, DSM_LOSS_THREADS, 0, s>>>((const float*)op.src0, (const float*)op.src1,
                                                         (double*)op.dst, op.C0, op.H * op.W,
                                                         op.Cout > 0 ? op.Cout : op.C0, (op.flags & MCVD_F_L1) ? 1 : 0);
  MCVD_CUDA_LAUNCH_CHECK("dsm_loss");
  return 0;
}

}  // namespace mcvd
