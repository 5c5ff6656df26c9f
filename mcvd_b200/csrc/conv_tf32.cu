// TF32 tensor-core convolutions of the FVD (I3D), FID (Inception-v3) and LPIPS (AlexNet) networks:
// MCVD_OP_CONV3D_TF32, MCVD_OP_CONV2D_TF32 and MCVD_OP_CONV_RELU_TF32 in include/mcvd_b200.h.  Same geometry, gather,
// epilogue and channel-slice output as MCVD_OP_CONV3D, MCVD_OP_CONV2D and MCVD_OP_CONV_RELU (conv_eval.cuh,
// conv_eval.cu); the products run on wgmma m64nNk8 tf32 with fp32 accumulators.
//
// Implicit GEMM: M = output positions (video * t * y * x, or frame * y * x), N = Cout, K = taps * Cin in
// (dt, dy, dx, c) order.  A CTA of two warpgroups computes a 128-position x BN tile; K advances in slabs of 32.
//   A (activations): every thread gathers its share of the slab's im2col rows as 16-byte chunks (Cin % 4 == 0, so a
//     chunk never straddles a tap; padding taps and K past the end are zero), rounds each value once to TF32 with
//     round-to-nearest (cvt.rna) and stores it into the K-major core-matrix layout wgmma reads.  The next slab's
//     loads are in flight while the current slab's wgmmas run.
//   B (weights): a packed image (mcvd_tf32_pack_weights) holds every (n tile, K slab) pair as one contiguous copy of
//     its shared-memory layout, already rounded to TF32, so it is staged with plain 16-byte cp.async.
// The tensor cores therefore never see a value with low mantissa bits set, and nothing depends on how they treat
// them.  Each output is one accumulator chain over K in slab order, with no split-K, so a video's or frame's
// features are the same bits whichever M tile, chunk or batch position it lands in.
#include "conv_eval.cuh"
#include "umma_ptx.cuh"

namespace mcvd {

using namespace ptx;

constexpr int TF_BM = 128;       // output positions per CTA: two consumer warpgroups of 64
constexpr int TF_BK = 32;        // K per slab: 8 core-matrix columns of 4 tf32
constexpr int TF_THREADS = 256;

// n tile for Cout: the width of {32, 64, 96, 128} with the smallest cost ntiles * (width + 64), where 64 stands for
// the A operand each n tile re-gathers and re-stages; ties go to the wider tile.  Shared by packing and launch.
static int tf32_ntile(int Cout) {
  int best = 128;
  long long best_cost = (long long)cdiv(Cout, 128) * (128 + 64);
  for (int bn = 96; bn >= 32; bn -= 32) {
    const long long cost = (long long)cdiv(Cout, bn) * (bn + 64);
    if (cost < best_cost) best = bn, best_cost = cost;
  }
  return best;
}

__device__ __forceinline__ float tf32_rna(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return __uint_as_float(r);
}

__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }

// Shared memory: two stages of A [32 k / 4][128 rows][4] and B [32 k / 4][BN cols][4], both the K-major no-swizzle
// core-matrix layout (8 rows x 16 bytes per core matrix, row groups 128 bytes apart, K columns of 4 a whole tile
// apart).  Thread roles: in the gather, warp w stages rows 8w .. 8w+7 and 64 + 8w .. 64 + 8w+7, lane l row 8w + l % 8
// and K columns l / 8 and 4 + l / 8 (a phase of 8 lanes stores 8 consecutive rows of one column: no bank conflicts;
// for 1x1 convs the 4 column lanes of a row read 64 contiguous bytes).  In the MMA, warpgroup wg owns rows
// 64 wg .. 64 wg + 63 of the tile.
template <int MODE, int BN>
__global__ void __launch_bounds__(TF_THREADS, 2)
    k_conv_tf32(const float* __restrict__ src, const float* __restrict__ wp, const float* __restrict__ bias,
                float* __restrict__ dst, ConvGeom g, int nk, int ntiles) {
  extern __shared__ __align__(128) float tf_smem[];
  constexpr int A_STAGE = TF_BM * TF_BK, B_STAGE = BN * TF_BK;    // floats
  float* As = tf_smem;
  float* Bs = tf_smem + 2 * A_STAGE;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int nt = (int)(blockIdx.x % (unsigned)ntiles);
  const long long m0 = (long long)(blockIdx.x / (unsigned)ntiles) * TF_BM;
  const int n0 = nt * BN;
  const int prow = 8 * warp + (lane & 7), pkc = lane >> 3;
  const ConvPos q[2] = {conv_pos<MODE>(src, g, m0 + prow), conv_pos<MODE>(src, g, m0 + prow + 64)};
  const float* wtile = wp + (long long)nt * nk * B_STAGE;
  const uint32_t as0 = smem_u32(As), bs0 = smem_u32(Bs);

  float4 ra[2][2];                                         // [K column j][row i] of the next slab
  auto load_a = [&](int kb) {
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const ConvTap t = conv_tap<MODE>(g, kb * TF_BK + 4 * (pkc + 4 * j));
#pragma unroll
      for (int i = 0; i < 2; ++i) ra[j][i] = conv_gather<MODE, true>(q[i], g, t);
    }
  };
  auto store_a = [&](int s) {
#pragma unroll
    for (int j = 0; j < 2; ++j)
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const float4 v = make_float4(tf32_rna(ra[j][i].x), tf32_rna(ra[j][i].y), tf32_rna(ra[j][i].z),
                                     tf32_rna(ra[j][i].w));
        *reinterpret_cast<float4*>(As + s * A_STAGE + ((pkc + 4 * j) * TF_BM + prow + 64 * i) * 4) = v;
      }
  };
  auto load_b = [&](int kb, int s) {
    const float* img = wtile + (long long)kb * B_STAGE;
#pragma unroll
    for (int c = tid; c < B_STAGE / 4; c += TF_THREADS)
      cp_async16(bs0 + (uint32_t)(s * B_STAGE + 4 * c) * 4u, img + 4 * c);
    cp_async_commit();
  };

  float acc[BN / 2];
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;

  load_a(0);
  load_b(0, 0);
  store_a(0);
  cp_async_wait_all();
  fence_proxy_async();                                     // generic-proxy stores -> the tensor cores' async proxy
  __syncthreads();

  const int wg = warp >> 2;
  const uint64_t a_proto = make_desc(0, TF_BM * 16, 128), b_proto = make_desc(0, BN * 16, 128);
  for (int kb = 0; kb < nk; ++kb) {
    const int s = kb & 1;
    const bool more = kb + 1 < nk;
    if (more) {                                            // the next slab's loads fly while this slab's MMAs run
      load_a(kb + 1);
      load_b(kb + 1, s ^ 1);
    }
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < TF_BK / 8; ++ks) {
      const uint64_t da = desc_add(a_proto, ((as0 + (uint32_t)(s * A_STAGE) * 4u) >> 4) + (uint32_t)(64 * wg) +
                                                (uint32_t)(2 * ks * TF_BM));
      const uint64_t db = desc_add(b_proto, ((bs0 + (uint32_t)(s * B_STAGE) * 4u) >> 4) + (uint32_t)(2 * ks * BN));
      wgmma_tf32<BN>(acc, da, db, 1);
    }
    wgmma_commit();
    if (more) store_a(s ^ 1);                              // stage s ^ 1 was last read by the previous slab's MMAs
    wgmma_wait<0>();
    cp_async_wait_all();
    fence_proxy_async();
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) reg_fence(acc[i]);

  // epilogue: thread owns rows r and r + 8 of its warp's 16, two adjacent columns of every 8-column block
  const int r0 = 64 * wg + 16 * (warp & 3) + (lane >> 2);
  const int cq = 2 * (lane & 3);
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
    const int n = n0 + 8 * j + cq;
    if (n0 + 8 * j >= g.Cout) break;                       // Cout % 8 == 0: an 8-column block is wholly in or out
    const float2 bv = __ldg(reinterpret_cast<const float2*>(bias + n));
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const long long m = m0 + r0 + 8 * i;
      if (m >= g.M) continue;
      float2 o;
      o.x = fmaxf(acc[4 * j + 2 * i] + bv.x, 0.f);
      o.y = fmaxf(acc[4 * j + 2 * i + 1] + bv.y, 0.f);
      *reinterpret_cast<float2*>(dst + m * g.pitch + g.off + n) = o;
    }
  }
}

// packed image: for every n tile, for every K slab, [8 K columns][BN][4] fp32 values rounded to TF32; K past the
// end and columns past Cout are zero
__global__ void __launch_bounds__(256) k_tf32_pack(const float* __restrict__ w, float* __restrict__ out, int K,
                                                   int Cout, int BN, int nk, long long total) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int stage = BN * TF_BK;
  const long long img = idx / stage;                       // nt * nk + kb
  const int e = (int)(idx - img * stage);
  const int nt = (int)(img / nk), kb = (int)(img - (long long)nt * nk);
  const int kc = e / (BN * 4), r = e - kc * BN * 4;
  const int n = nt * BN + r / 4, k = kb * TF_BK + kc * 4 + (r & 3);
  out[idx] = (k < K && n < Cout) ? tf32_rna(w[(long long)k * Cout + n]) : 0.f;
}

static long long tf32_packed_floats(int K, int Cout) {
  if (K < 1 || Cout < 8 || Cout % 8) return -1;
  const int bn = tf32_ntile(Cout);
  return (long long)cdiv(K, TF_BK) * TF_BK * cdiv(Cout, bn) * bn;
}

const char* conv_tf32_geom(const McvdOp& op, ConvGeom& g) {
  if (const char* why = conv_geom(op, g)) return why;
  if ((g.M + TF_BM - 1) / TF_BM * cdiv(op.Cout, tf32_ntile(op.Cout)) > 0x7fffffffLL)
    return "too many output positions for the grid";
  return nullptr;
}

template <int MODE, int BN>
static int run_tf32(const McvdOp& op, const ConvGeom& g, cudaStream_t s) {
  const size_t smem = (size_t)2 * (TF_BM + BN) * TF_BK * sizeof(float);
  cudaError_t e = cudaFuncSetAttribute(k_conv_tf32<MODE, BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  MCVD_CHECK(e == cudaSuccess, "CONV_TF32: cudaFuncSetAttribute failed: %s", cudaGetErrorString(e));
  const int ntiles = cdiv(g.Cout, BN);
  const long long ctas = (g.M + TF_BM - 1) / TF_BM * ntiles;
  k_conv_tf32<MODE, BN><<<(unsigned)ctas, TF_THREADS, smem, s>>>((const float*)op.src0, (const float*)op.w,
                                                                (const float*)op.bias, (float*)op.dst, g,
                                                                cdiv(g.K, TF_BK), ntiles);
  MCVD_CUDA_LAUNCH_CHECK("conv_tf32");
  return 0;
}

template <int MODE>
static int run_tf32_mode(const McvdOp& op, const ConvGeom& g, cudaStream_t s) {
  switch (tf32_ntile(g.Cout)) {
    case 32: return run_tf32<MODE, 32>(op, g, s);
    case 64: return run_tf32<MODE, 64>(op, g, s);
    case 96: return run_tf32<MODE, 96>(op, g, s);
    default: return run_tf32<MODE, 128>(op, g, s);
  }
}

int launch_conv_tf32(const McvdOp& op, cudaStream_t s) {
  // the AlexNet geometry leaves the input and output pointers to this check, as launch_conv_ffma does
  if (op.kind == MCVD_OP_CONV_RELU_TF32) MCVD_CHECK(op.src0 && op.dst, "%s: null pointer", conv_kind_name(op.kind));
  ConvGeom g;
  if (const char* why = conv_tf32_geom(op, g)) MCVD_CHECK(false, "%s: %s", conv_kind_name(op.kind), why);
  // G_S2MAX keeps its 3x3 window unrolled: at 128 registers it still fits two CTAs per SM without spilling
  switch (gather_mode(op)) {
    case G_CONV2: return run_tf32_mode<G_CONV2>(op, g, s);
    case G_CONV3: return run_tf32_mode<G_CONV3>(op, g, s);
    case G_PW: return run_tf32_mode<G_PW>(op, g, s);
    case G_BMAX: return run_tf32_mode<G_BMAX>(op, g, s);
    case G_BAVG: return run_tf32_mode<G_BAVG>(op, g, s);
    default: return run_tf32_mode<G_S2MAX>(op, g, s);
  }
}

}  // namespace mcvd

extern "C" {

long long mcvd_tf32_packed_bytes(int K, int Cout) {
  const long long n = mcvd::tf32_packed_floats(K, Cout);
  if (n < 0) {
    mcvd::set_error("tf32 packing: K = %d, Cout = %d (K >= 1, Cout a positive multiple of 8)", K, Cout);
    return -1;
  }
  return n * (long long)sizeof(float);
}

int mcvd_tf32_pack_weights(const float* w_kmajor, int K, int Cout, void* out, void* stream) {
  const long long total = mcvd::tf32_packed_floats(K, Cout);
  if (total < 0) {
    mcvd::set_error("tf32 packing: K = %d, Cout = %d (K >= 1, Cout a positive multiple of 8)", K, Cout);
    return -1;
  }
  if (!w_kmajor || !out || (reinterpret_cast<uintptr_t>(out) & 15)) {
    mcvd::set_error("tf32 packing: null weights, or output null or not 16-byte aligned");
    return -1;
  }
  const int bn = mcvd::tf32_ntile(Cout);
  mcvd::k_tf32_pack<<<(unsigned)((total + 255) / 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      w_kmajor, (float*)out, K, Cout, bn, mcvd::cdiv(K, mcvd::TF_BK), total);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    mcvd::set_error("tf32 packing: launch failed: %s", cudaGetErrorString(e));
    return -2;
  }
  return 0;
}

}  // extern "C"
