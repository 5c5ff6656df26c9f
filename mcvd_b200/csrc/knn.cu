// k-nearest-neighbour precision / recall of two feature sets without the distance matrix: see MCVD_OP_KNN_RADIUS and
// MCVD_OP_KNN_COVER in include/mcvd_b200.h.  A distance is sqrtf of the fp32 sum over d = 0 .. D-1, in that order,
// of (a_d - b_d)^2 (one subtract and one FMA per term), so the same pair gives the same bits in every pass and a
// point's distance to itself is exactly 0.
//
// Tiling (the FFMA tile of k_conv_ffma, conv_eval.cu): one CTA owns 64 rows of A and streams B past them in 64-row tiles,
// 16 features deep, the next slice prefetched into registers; each thread holds a 4 x 4 block of squared distances.
// After each B tile a thread folds its 16 distances into per-row state held in registers:
//   RADIUS: the 8 smallest squared distances of each of its 4 rows over the columns it has seen (sorted, with
//           multiplicity, so ties count as torch.kthvalue counts them); at the end the 16 threads that share rows
//           merge their lists with warp shuffles and the rank-th smallest is the radius.
//   COVER:  whether any column b of the tile has d(a, b) <= radius_b; a CTA stops streaming once all its rows are
//           covered.
// State is O(rows); nothing of size Na x Nb is stored.
#include <math.h>

#include "mcvd_common.cuh"

namespace mcvd {

constexpr int KN_BM = 64, KN_BN = 64, KN_BK = 16, KN_MAXR = 8;

// insert v into the ascending list L (the largest value drops out)
__device__ __forceinline__ void knn_insert(float (&L)[KN_MAXR], float v) {
#pragma unroll
  for (int j = 0; j < KN_MAXR; ++j) {
    const float lo = fminf(L[j], v);
    v = fmaxf(L[j], v);
    L[j] = lo;
  }
}

// one 16-deep slice of 64 rows of X [N, D] starting at row r0: thread (row tid % 64, features 4 * (tid / 64) ..)
__device__ __forceinline__ float4 knn_load(const float* __restrict__ X, int N, int D, int r0, int k) {
  const int r = r0 + threadIdx.x % KN_BM;
  if (r >= N || k >= D) return make_float4(0.f, 0.f, 0.f, 0.f);    // zero pairs add exactly 0 to a sum
  return *reinterpret_cast<const float4*>(X + (long long)r * D + k);
}

template <bool COVER>
__global__ void __launch_bounds__(256, COVER ? 2 : 1) k_knn(const float* __restrict__ A, const float* __restrict__ B,
                                                const float* __restrict__ radii, int Na, int Nb, int D, int rank,
                                                float* __restrict__ rad_out, int* __restrict__ flag_out) {
  __shared__ __align__(16) float As[2][KN_BK][KN_BM];
  __shared__ __align__(16) float Bs[2][KN_BK][KN_BN];
  __shared__ int covered[KN_BM];
  const int tid = threadIdx.x;
  const int m0 = blockIdx.x * KN_BM;
  const int lm = tid % KN_BM, lk = (tid / KN_BM) * 4;
  const int tm = (tid / 16) * 4, tn = (tid % 16) * 4;
  const int slices = (D + KN_BK - 1) / KN_BK;
  const int tiles = (Nb + KN_BN - 1) / KN_BN;
  const long long steps = (long long)slices * tiles;
  float L[4][KN_MAXR];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < KN_MAXR; ++j) L[i][j] = INFINITY;
  if (COVER && tid < KN_BM) covered[tid] = m0 + tid >= Na;
  float acc[4][4] = {};
  float4 ra = knn_load(A, Na, D, m0, lk);
  float4 rb = knn_load(B, Nb, D, 0, lk);
  int buf = 0;
  for (long long st = 0; st < steps; ++st) {
    const int tile = (int)(st / slices), slice = (int)(st - (long long)tile * slices);
    As[buf][lk + 0][lm] = ra.x; As[buf][lk + 1][lm] = ra.y; As[buf][lk + 2][lm] = ra.z; As[buf][lk + 3][lm] = ra.w;
    Bs[buf][lk + 0][lm] = rb.x; Bs[buf][lk + 1][lm] = rb.y; Bs[buf][lk + 2][lm] = rb.z; Bs[buf][lk + 3][lm] = rb.w;
    __syncthreads();
    if (st + 1 < steps) {
      const int nt = slice + 1 < slices ? tile : tile + 1, ns = slice + 1 < slices ? slice + 1 : 0;
      ra = knn_load(A, Na, D, m0, ns * KN_BK + lk);
      rb = knn_load(B, Nb, D, nt * KN_BN, ns * KN_BK + lk);
    }
#pragma unroll
    for (int kk = 0; kk < KN_BK; ++kk) {
      const float4 a = *reinterpret_cast<const float4*>(&As[buf][kk][tm]);
      const float4 b = *reinterpret_cast<const float4*>(&Bs[buf][kk][tn]);
      const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float d = av[i] - bv[j];
          acc[i][j] = fmaf(d, d, acc[i][j]);
        }
    }
    buf ^= 1;                                      // the other buffer was last read before this slice's barrier
    if (slice + 1 < slices) continue;
    // the tile's distances are complete: fold them into the row state and start the next tile from zero
    const int n0 = tile * KN_BN + tn;
    bool hit[4] = {false, false, false, false};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const bool col = n0 + j < Nb;
      const float r = COVER && col ? radii[n0 + j] : 0.f;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        if (COVER) hit[i] |= col && sqrtf(acc[i][j]) <= r;
        else knn_insert(L[i], col ? acc[i][j] : INFINITY);
      }
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      if (COVER && hit[i]) covered[tm + i] = 1;
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
    }
    if (COVER && __syncthreads_and(tid >= KN_BM || covered[tid])) break;   // every row of the CTA is covered
  }
  if constexpr (COVER) {
    __syncthreads();
    if (tid < KN_BM && m0 + tid < Na) flag_out[m0 + tid] = covered[tid];
  } else {
    // the 16 threads of a row group are lanes 0-15 or 16-31 of one warp: butterfly-merge their lists
#pragma unroll
    for (int step = 0; step < 4; ++step)
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        float other[KN_MAXR];
#pragma unroll
        for (int j = 0; j < KN_MAXR; ++j) other[j] = __shfl_xor_sync(0xffffffffu, L[i][j], 8 >> step);
#pragma unroll
        for (int j = 0; j < KN_MAXR; ++j) knn_insert(L[i], other[j]);
      }
    if (tid % 16) return;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float v = L[i][0];
#pragma unroll
      for (int j = 1; j < KN_MAXR; ++j)
        if (j == rank - 1) v = L[i][j];
      if (m0 + tm + i < Na) rad_out[m0 + tm + i] = sqrtf(v);
    }
  }
}

const char* knn_error(const McvdOp& op) {
  if (!op.src0 || !op.src1 || !op.dst) return "null features or output";
  if (op.kind == MCVD_OP_KNN_COVER && !op.aux0) return "null radii";
  if (op.C0 <= 0 || op.C0 % 4) return "feature size must be a positive multiple of 4";
  if (op.i0 < 1) return "second set is empty";
  if (op.H != 1 || op.W != 1) return "output size must be 1x1";
  if (op.kind == MCVD_OP_KNN_RADIUS && (op.i1 < 1 || op.i1 > KN_MAXR)) return "rank must be in 1 .. 8";
  if (op.kind == MCVD_OP_KNN_RADIUS && op.i1 > op.i0) return "rank larger than the second set";
  if (op.flags) return "no flags are defined for the k-NN kinds";
  return nullptr;
}

int launch_knn(const McvdOp& op, cudaStream_t s) {
  const bool cover = op.kind == MCVD_OP_KNN_COVER;
  if (const char* why = knn_error(op)) MCVD_CHECK(false, "%s: %s", cover ? "KNN_COVER" : "KNN_RADIUS", why);
  const unsigned grid = (unsigned)cdiv(op.B, KN_BM);
  if (cover)
    k_knn<true><<<grid, 256, 0, s>>>((const float*)op.src0, (const float*)op.src1, (const float*)op.aux0, op.B, op.i0,
                                     op.C0, 0, nullptr, (int*)op.dst);
  else
    k_knn<false><<<grid, 256, 0, s>>>((const float*)op.src0, (const float*)op.src1, nullptr, op.B, op.i0, op.C0,
                                      op.i1, (float*)op.dst, nullptr);
  MCVD_CUDA_LAUNCH_CHECK(cover ? "knn_cover" : "knn_radius");
  return 0;
}

}  // namespace mcvd
