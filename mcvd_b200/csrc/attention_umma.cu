// Multi-head self-attention over the H*W tokens of a sample on the Hopper tensor cores (wgmma), flash style
// (reference AttnBlockpp.forward, models/better/layerspp.py:239-245: w = softmax_j(q_i.k_j * Ch^-0.5),
// h_i = sum_j w_ij v_j; the reference materialises w as [B*heads, HW, HW] fp32).
//
//   qkv [B, T, 3C] fp32 (q | k | v along channels; head h = channels [h*d, (h+1)*d)),  out [B, T, C]
//   grid = (ceil(T / 128), heads, B); one CTA owns 128 query rows and walks the keys in tiles of KT.
//
// Per key tile, each of the two consumer warpgroups (64 query rows):
//                 S = Q K^T   (wgmma m64nKTk16, both operands from shared memory)   -> registers
//                 P = exp(S*scale - m), online max / sum in registers (a row lives in the 4 lanes of a quad)
//                 O = O * exp(m_old - m_new) + P V   (wgmma m64nDk16, P from registers: the fp32 accumulator
//                     layout of S is the register A-operand layout, so P never touches shared memory; wgmma's
//                     N stops at 256, so head dim 288 issues it as two N = 144 halves of the channels)
// fp32 parity: q, k, v and p are split into fp16 hi + lo and every product is 3 MMAs
// (hi*hi + lo*hi + hi*lo), fp32 accumulation -- same scheme as conv_umma.cu.
//
// Operand layouts (canonical K-major, no swizzle): [k-chunk of 8 halfs][row][16 B], LBO = rows*16,
// SBO = 128.   V is staged transposed (rows = channels, k = keys) so it is K-major too.
//
// Two launches per op:
//   k_attn_presplit  converts q, k, v ONCE into fp16 hi/lo "operand images" in a scratch buffer, one image per
//                    (sample, head, tile), byte-for-byte what the MMA wants in shared memory (converting inside
//                    the attention kernel would redo the K/V tiles for each of the T/128 query tiles).
//   k_attention_umma one thread streams the images in with cp.async.bulk (mbarrier complete_tx).
#include "mcvd_common.cuh"
#include "umma_ptx.cuh"

namespace mcvd {

namespace {

using namespace ptx;

constexpr int QT = 128;
constexpr int ATT_THREADS = 288;       // 2 consumer warpgroups + image loader
// Head dims 256 / 288 hold 128 / 144 O accumulators per consumer thread, more than the 168 registers a 288- or
// 384-thread CTA gets.  There the loader is a whole warpgroup that hands registers to the consumers (setmaxnreg):
// 2 x 128 x 232 + 128 x 40 <= 64 K.
template <int D> __host__ __device__ constexpr bool wide_head() { return D > 192; }
template <int D> __host__ __device__ constexpr int att_threads() { return wide_head<D>() ? 384 : ATT_THREADS; }
constexpr int REG_LOAD_WIDE = 40, REG_CONS_WIDE = 232;
constexpr int SPLIT_THREADS = 256;

struct AttnArgs {
  const float* qkv;
  float* out;
  uint8_t* img;                 // operand images: [Q tiles | K tiles | V tiles], see image_offsets()
  long long k_off, v_off;       // byte offsets of the K and V image arrays
  int T, C, KT, nkt, nqt, nst;
  float scale;
};

// fp32 x8 -> fp16 hi (16 B) + lo (16 B)
__device__ __forceinline__ void split8(const float v[8], uint4& hv, uint4& lv) {
  uint32_t hw[4], lw[4];
#pragma unroll
  for (int e = 0; e < 4; ++e) split2(v[2 * e], v[2 * e + 1], hw[e], lw[e]);
  hv = make_uint4(hw[0], hw[1], hw[2], hw[3]);
  lv = make_uint4(lw[0], lw[1], lw[2], lw[3]);
}

// stage `rows` token rows x D channels (channel-contiguous in global) as a K-major operand
//   dst[(c8 * rows + r) * 16]  <-  src[(row0 + r) * stride + c8 * 8 .. +8)
template <int D>
__device__ __forceinline__ void stage_rows(uint8_t* hi, uint8_t* lo, const float* src, long long stride, int rows,
                                           int valid_rows, int tid, int nthreads) {
  constexpr int U = 6;                                   // units in flight per thread (12 x LDG.128)
  const int units = (D / 8) * rows;
  for (int u0 = tid; u0 < units; u0 += nthreads * U) {
    float4 va[U], vb[U];
#pragma unroll
    for (int i = 0; i < U; ++i) {
      const int u = u0 + i * nthreads;
      const int c8 = u / rows, r = u - c8 * rows;
      va[i] = vb[i] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (u < units && r < valid_rows) {
        const float4* p = reinterpret_cast<const float4*>(src + (long long)r * stride + c8 * 8);
        va[i] = __ldg(p);
        vb[i] = __ldg(p + 1);
      }
    }
#pragma unroll
    for (int i = 0; i < U; ++i) {
      const int u = u0 + i * nthreads;
      if (u < units) {
        const int c8 = u / rows, r = u - c8 * rows;
        const float v[8] = {va[i].x, va[i].y, va[i].z, va[i].w, vb[i].x, vb[i].y, vb[i].z, vb[i].w};
        uint4 hv, lv;
        split8(v, hv, lv);
        const size_t off = ((size_t)c8 * rows + r) * 16;
        *reinterpret_cast<uint4*>(hi + off) = hv;
        *reinterpret_cast<uint4*>(lo + off) = lv;
      }
    }
  }
}

// V^T image: rows = channels, k = keys.  unit = (key chunk kc of 8 keys, 4 channels): 8 x LDG.128 (one per
// key, 4 channels each), transposed in registers into 4 rows of 8 keys; 2 units (16 loads) in flight.
template <int D>
__device__ __forceinline__ void stage_v(uint8_t* vh, uint8_t* vl, const float* vsrc, long long stride, int KT, int tid,
                                        int nthreads) {
  constexpr int C4 = D / 4;
  const int vunits = (KT / 8) * C4;
  for (int u0 = tid; u0 < vunits; u0 += 2 * nthreads) {
    float4 ld[2][8];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int u = u0 + i * nthreads;
      const int kc = u / C4, c4 = u - kc * C4;
#pragma unroll
      for (int e = 0; e < 8; ++e)
        ld[i][e] = (u < vunits) ? __ldg(reinterpret_cast<const float4*>(vsrc + (long long)(kc * 8 + e) * stride) + c4)
                                : make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int u = u0 + i * nthreads;
      if (u < vunits) {
        const int kc = u / C4, c4 = u - kc * C4;
        const float r0[8] = {ld[i][0].x, ld[i][1].x, ld[i][2].x, ld[i][3].x, ld[i][4].x, ld[i][5].x, ld[i][6].x, ld[i][7].x};
        const float r1[8] = {ld[i][0].y, ld[i][1].y, ld[i][2].y, ld[i][3].y, ld[i][4].y, ld[i][5].y, ld[i][6].y, ld[i][7].y};
        const float r2[8] = {ld[i][0].z, ld[i][1].z, ld[i][2].z, ld[i][3].z, ld[i][4].z, ld[i][5].z, ld[i][6].z, ld[i][7].z};
        const float r3[8] = {ld[i][0].w, ld[i][1].w, ld[i][2].w, ld[i][3].w, ld[i][4].w, ld[i][5].w, ld[i][6].w, ld[i][7].w};
        uint4 hv, lv;
        const size_t off = ((size_t)kc * D + c4 * 4) * 16;
        split8(r0, hv, lv); *reinterpret_cast<uint4*>(vh + off) = hv;      *reinterpret_cast<uint4*>(vl + off) = lv;
        split8(r1, hv, lv); *reinterpret_cast<uint4*>(vh + off + 16) = hv; *reinterpret_cast<uint4*>(vl + off + 16) = lv;
        split8(r2, hv, lv); *reinterpret_cast<uint4*>(vh + off + 32) = hv; *reinterpret_cast<uint4*>(vl + off + 32) = lv;
        split8(r3, hv, lv); *reinterpret_cast<uint4*>(vh + off + 48) = hv; *reinterpret_cast<uint4*>(vl + off + 48) = lv;
      }
    }
  }
}

// key tile: as large as the operand images allow in shared memory (Q is resident: 4*D*128 bytes).  Head dims 256
// and 288 (128 / 144 KiB of Q) fit one K + V^T stage of 32 keys (64 / 72 KiB), not two: see launch_d.
template <int D> __host__ __device__ constexpr int kt_max() { return D <= 96 ? 128 : (D <= 128 ? 64 : 32); }

// the key tile a T-token attention runs with (T itself when smaller than kt_max), 0 when T is not a whole number
// of key tiles the kernel is built for.  The lowering asks for it through mcvd_attention_key_tile.
template <int D> int key_tile(int T) {
  const int kt = T < kt_max<D>() ? T : kt_max<D>();
  return ((kt == 32 || kt == 64 || kt == 128) && T % kt == 0) ? kt : 0;
}

// image sizes in bytes (hi plane + lo plane)
template <int D> __host__ __device__ constexpr long long q_image_bytes() { return 2LL * (D / 8) * QT * 16; }
template <int D> __host__ __device__ inline long long kv_image_bytes(int KT) { return 2LL * (D / 8) * KT * 16; }

// Pre-pass: grid (nqt + 2 nkt, heads, B); block x builds one Q, K or V image of (sample, head).
template <int D>
__global__ void __launch_bounds__(SPLIT_THREADS) k_attn_presplit(const AttnArgs a) {
  const int x = blockIdx.x, h = blockIdx.y, b = blockIdx.z, heads = gridDim.y;
  const int C3 = 3 * a.C, KT = a.KT;
  const float* base = a.qkv + (long long)b * a.T * C3 + h * D;
  const long long bh = (long long)b * heads + h;
  if (x < a.nqt) {
    uint8_t* dst = a.img + (bh * a.nqt + x) * q_image_bytes<D>();
    const int q0 = x * QT;
    stage_rows<D>(dst, dst + q_image_bytes<D>() / 2, base + (long long)q0 * C3, C3, QT, min(QT, a.T - q0), threadIdx.x,
                  SPLIT_THREADS);
  } else if (x < a.nqt + a.nkt) {
    const int kt = x - a.nqt;
    uint8_t* dst = a.img + a.k_off + (bh * a.nkt + kt) * kv_image_bytes<D>(KT);
    stage_rows<D>(dst, dst + kv_image_bytes<D>(KT) / 2, base + a.C + (long long)kt * KT * C3, C3, KT, KT, threadIdx.x,
                  SPLIT_THREADS);
  } else {
    const int kt = x - a.nqt - a.nkt;
    uint8_t* dst = a.img + a.v_off + (bh * a.nkt + kt) * kv_image_bytes<D>(KT);
    stage_v<D>(dst, dst + kv_image_bytes<D>(KT) / 2, base + 2 * a.C + (long long)kt * KT * C3, C3, KT, threadIdx.x,
               SPLIT_THREADS);
  }
}

// O += P V over one 16-key step: head dims up to 256 in one wgmma, 288 as two N = 144 halves (V^T rows =
// channels at 16 B, so the second half starts D/2 rows in; its accumulators are o[D/4 ..)).  Every output
// element still sums the same products in the same order.
template <int D>
__device__ __forceinline__ void wgmma_pv(float* o, const uint32_t* p, uint64_t v) {
  if constexpr (D <= 256) {
    wgmma_rs<D>(o, p, v);
  } else {
    wgmma_rs<D / 2>(o, p, v);
    wgmma_rs<D / 2>(o + D / 4, p, desc_add(v, D / 2));
  }
}

// Attention kernel: grid (nqt, heads, B), att_threads<D>() threads.  Warps 0-7 = two consumer warpgroups (query
// rows [64 wg, 64 wg + 64) of the tile), warp 8 = image loader (Q once, then K / V^T tiles through NST stages);
// warps 9-11 (wide heads only) just give their registers away.
template <int D, int KT>
__global__ void __launch_bounds__(att_threads<D>(), 1) k_attention_umma(const AttnArgs a) {
  constexpr bool WIDE = wide_head<D>();
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  constexpr int NQ = QT / 64;                 // consumer warpgroups
  const int NST = a.nst;
  const uint32_t q_bytes = (uint32_t)q_image_bytes<D>(), kv_bytes = (uint32_t)kv_image_bytes<D>(KT);
  uint8_t* qimg = smem_raw;                   // hi | lo
  uint8_t* kimg = qimg + q_bytes;             // [NST] hi | lo
  uint8_t* vimg = kimg + (size_t)NST * kv_bytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(vimg + (size_t)NST * kv_bytes);
  const uint32_t bar0 = smem_u32(bars);
  const uint32_t Q_FULL = bar0;
  auto K_FULL = [&](int i) { return bar0 + 8u * (1 + i); };
  auto V_FULL = [&](int i) { return bar0 + 8u * (3 + i); };
  auto K_EMPTY = [&](int i) { return bar0 + 8u * (5 + i); };
  auto V_EMPTY = [&](int i) { return bar0 + 8u * (7 + i); };

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int q0 = blockIdx.x * QT, h = blockIdx.y, b = blockIdx.z;
  const long long bh = (long long)b * gridDim.y + h;

  if (tid == 0) {
    mbar_init(Q_FULL, 1);
    for (int i = 0; i < 2; ++i) {
      mbar_init(K_FULL(i), 1); mbar_init(V_FULL(i), 1);
      mbar_init(K_EMPTY(i), 4 * NQ); mbar_init(V_EMPTY(i), 4 * NQ);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (WIDE ? warp >= 4 * NQ : warp == 4 * NQ) {
    // ================= image loader =================
    if constexpr (WIDE) setmaxnreg_dec<REG_LOAD_WIDE>();
    if ((!WIDE || warp == 4 * NQ) && elect_one()) {
      mbar_arrive_expect_tx(Q_FULL, q_bytes);
      bulk_g2s(smem_u32(qimg), a.img + (bh * a.nqt + blockIdx.x) * q_image_bytes<D>(), q_bytes, Q_FULL);
      for (int kt = 0; kt < a.nkt; ++kt) {
        const int st = kt % NST;
        const uint32_t ph = ((kt / NST) & 1) ^ 1;
        const long long off = (bh * a.nkt + kt) * kv_image_bytes<D>(KT);
        mbar_wait(K_EMPTY(st), ph);
        mbar_arrive_expect_tx(K_FULL(st), kv_bytes);
        bulk_g2s(smem_u32(kimg + (size_t)st * kv_bytes), a.img + a.k_off + off, kv_bytes, K_FULL(st));
        mbar_wait(V_EMPTY(st), ph);
        mbar_arrive_expect_tx(V_FULL(st), kv_bytes);
        bulk_g2s(smem_u32(vimg + (size_t)st * kv_bytes), a.img + a.v_off + off, kv_bytes, V_FULL(st));
      }
    }
    __syncwarp();
    return;
  }

  // ================= consumers: S = Q K^T, online softmax, O += P V =================
  if constexpr (WIDE) setmaxnreg_inc<REG_CONS_WIDE>();
  const int wg = warp >> 2, wq = warp & 3;
  const int r0 = 64 * wg + 16 * wq + (lane >> 2);          // query rows r0 and r0 + 8 of the tile
  const int cq = 2 * (lane & 3);
  // descriptors: Q rows at 16 B, K-chunks QT*16 apart; K tile rows (keys) at 16 B, chunks KT*16 apart;
  // V^T rows (channels) at 16 B, key chunks D*16 apart
  const uint64_t q_desc = make_desc(smem_u32(qimg) + 64u * 16u * wg, QT * 16, 128);
  const uint32_t q_lo16 = q_bytes / 32;                      // lo plane offset, 16-byte units
  const uint32_t kv_lo16 = kv_bytes / 32;
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
  float o[D / 2];
#pragma unroll
  for (int i = 0; i < D / 2; ++i) o[i] = 0.f;
  mbar_wait(Q_FULL, 0);
  for (int kt = 0; kt < a.nkt; ++kt) {
    const int st = kt % NST;
    const uint32_t ph = (kt / NST) & 1;
    float sacc[KT / 2];
    const uint64_t k_desc = make_desc(smem_u32(kimg + (size_t)st * kv_bytes), KT * 16, 128);
    mbar_wait(K_FULL(st), ph);
    wgmma_fence();
#pragma unroll
    for (int s = 0; s < D / 16; ++s) {
      const uint64_t qh = desc_add(q_desc, 2u * s * QT), ql = desc_add(qh, q_lo16);
      const uint64_t kh = desc_add(k_desc, 2u * s * KT), kl = desc_add(kh, kv_lo16);
      wgmma_ss<KT>(sacc, qh, kh, s);
      wgmma_ss<KT>(sacc, ql, kh, 1);
      wgmma_ss<KT>(sacc, qh, kl, 1);
    }
    wgmma_commit();
    wgmma_wait<0>();
#pragma unroll
    for (int i = 0; i < KT / 2; ++i) reg_fence(sacc[i]);
    if (lane == 0) mbar_arrive(K_EMPTY(st));
    // online softmax: a query row lives in the 4 lanes of a quad
    float alpha[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      float mx = -INFINITY;
#pragma unroll
      for (int j = 0; j < KT / 8; ++j)
        mx = fmaxf(mx, fmaxf(sacc[4 * j + 2 * i], sacc[4 * j + 2 * i + 1]));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float mn = fmaxf(m[i], mx * a.scale);
      alpha[i] = expf(m[i] - mn);
      m[i] = mn;
      float sum = 0.f;
#pragma unroll
      for (int j = 0; j < KT / 8; ++j) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const float p = expf(fmaf(sacc[4 * j + 2 * i + e], a.scale, -mn));
          sacc[4 * j + 2 * i + e] = p;
          sum += p;
        }
      }
      l[i] = l[i] * alpha[i] + sum;
    }
#pragma unroll
    for (int j = 0; j < D / 8; ++j) {
      o[4 * j] *= alpha[0]; o[4 * j + 1] *= alpha[0];
      o[4 * j + 2] *= alpha[1]; o[4 * j + 3] *= alpha[1];
    }
    // P (fp16 hi / lo pairs in the accumulator layout == the register A-operand layout of m64nNk16)
    const uint64_t v_desc = make_desc(smem_u32(vimg + (size_t)st * kv_bytes), D * 16, 128);
    mbar_wait(V_FULL(st), ph);
    uint32_t ph4[KT / 16][4], pl4[KT / 16][4];
#pragma unroll
    for (int kk = 0; kk < KT / 16; ++kk)
#pragma unroll
      for (int r = 0; r < 4; ++r) split2(sacc[8 * kk + 2 * r], sacc[8 * kk + 2 * r + 1], ph4[kk][r], pl4[kk][r]);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < KT / 16; ++kk) {
      const uint64_t vh = desc_add(v_desc, 2u * kk * D), vl = desc_add(vh, kv_lo16);
      wgmma_pv<D>(o, ph4[kk], vh);
      wgmma_pv<D>(o, pl4[kk], vh);
      wgmma_pv<D>(o, ph4[kk], vl);
    }
    wgmma_commit();
    wgmma_wait<0>();
#pragma unroll
    for (int i = 0; i < D / 2; ++i) reg_fence(o[i]);
    if (lane == 0) mbar_arrive(V_EMPTY(st));
  }
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    l[i] += __shfl_xor_sync(0xffffffffu, l[i], 1);
    l[i] += __shfl_xor_sync(0xffffffffu, l[i], 2);
  }
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int q = q0 + r0 + 8 * i;
    if (q >= a.T) continue;
    const float inv = 1.0f / l[i];
    float* orow = a.out + ((long long)b * a.T + q) * a.C + h * D;
#pragma unroll
    for (int j = 0; j < D / 8; ++j)
      *reinterpret_cast<float2*>(orow + 8 * j + cq) = make_float2(o[4 * j + 2 * i] * inv, o[4 * j + 2 * i + 1] * inv);
  }
}

template <int D, int KT>
int launch_dk(const AttnArgs& a, size_t smem, const McvdOp& op, cudaStream_t s) {
  cudaError_t e = cudaFuncSetAttribute(k_attention_umma<D, KT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  MCVD_CHECK(e == cudaSuccess, "ATTENTION_UMMA: cudaFuncSetAttribute failed: %s", cudaGetErrorString(e));
  dim3 sgrid(a.nqt + 2 * a.nkt, op.i0, op.B);
  k_attn_presplit<D><<<sgrid, SPLIT_THREADS, 0, s>>>(a);
  MCVD_CUDA_LAUNCH_CHECK("attention presplit");
  dim3 grid(a.nqt, op.i0, op.B);
  k_attention_umma<D, KT><<<grid, att_threads<D>(), smem, s>>>(a);
  MCVD_CUDA_LAUNCH_CHECK("attention_umma");
  return 0;
}

template <int D>
int launch_d(const McvdOp& op, cudaStream_t s) {
  AttnArgs a;
  a.qkv = (const float*)op.src0; a.out = (float*)op.dst;
  a.T = op.H * op.W; a.C = op.C0; a.scale = op.f0;
  a.KT = key_tile<D>(a.T);
  MCVD_CHECK(a.KT > 0, "ATTENTION_UMMA: %d tokens not tileable by the key tile %d", a.T, min(a.T, kt_max<D>()));
  a.nkt = a.T / a.KT;
  a.nqt = cdiv(a.T, QT);
  a.img = (uint8_t*)op.dst2;
  const long long bh = (long long)op.B * op.i0;
  a.k_off = bh * a.nqt * q_image_bytes<D>();
  a.v_off = a.k_off + bh * a.nkt * kv_image_bytes<D>(a.KT);
  MCVD_CHECK(op.dst2, "ATTENTION_UMMA: dst2 (operand-image scratch, mcvd_attention_scratch_bytes) is NULL");
  MCVD_CHECK((reinterpret_cast<uintptr_t>(op.dst2) & 15) == 0, "ATTENTION_UMMA: scratch must be 16-byte aligned");
  // Q stays resident; K and V^T tiles are double-buffered when two stages fit (head dims up to 192).  At 256 / 288
  // one stage: the loader refills K while the consumers run the softmax and P V, and V^T while they run the next S.
  const size_t q_bytes = (size_t)q_image_bytes<D>(), kv_bytes = (size_t)kv_image_bytes<D>(a.KT);
  a.nst = (q_bytes + 4 * kv_bytes + 128 <= 227 * 1024) ? 2 : 1;
  const size_t smem = q_bytes + 2 * a.nst * kv_bytes + 128;
  MCVD_CHECK(smem <= 227 * 1024, "ATTENTION_UMMA: %zu B of shared memory", smem);
  // key tiles never exceed kt_max<D>() (the S registers and shared memory are sized for it)
  if (a.KT == 32) return launch_dk<D, 32>(a, smem, op, s);
  if (a.KT == 64) return launch_dk<D, (kt_max<D>() >= 64 ? 64 : 32)>(a, smem, op, s);
  return launch_dk<D, kt_max<D>()>(a, smem, op, s);
}

}  // namespace

// bytes of operand-image scratch an ATTENTION_UMMA op needs: Q padded to whole 128-row tiles, K and V
// exactly T rows; fp16 hi + lo = 4 bytes per element
long long attention_umma_scratch_bytes(int B, int T, int C) {
  if (B <= 0 || T <= 0 || C <= 0) return 0;
  return 4LL * B * C * ((long long)cdiv(T, QT) * QT + 2LL * T);
}

// the head dims the kernel is built for, with the key tile of T tokens (0: not built for d, or T not tileable)
int attention_umma_key_tile(int T, int d) {
  if (T <= 0) return 0;
  switch (d) {
    case 32: return key_tile<32>(T);
    case 48: return key_tile<48>(T);
    case 64: return key_tile<64>(T);
    case 96: return key_tile<96>(T);
    case 128: return key_tile<128>(T);
    case 192: return key_tile<192>(T);
    case 256: return key_tile<256>(T);
    case 288: return key_tile<288>(T);
    default: return 0;
  }
}

int launch_attention_umma(const McvdOp& op, cudaStream_t s) {
  MCVD_CHECK(op.src0 && op.dst, "ATTENTION_UMMA: null pointer");
  MCVD_CHECK(op.i0 * op.i1 == op.C0, "ATTENTION_UMMA: heads %d x dim %d != channels %d", op.i0, op.i1, op.C0);
  switch (op.i1) {
    case 32: return launch_d<32>(op, s);
    case 48: return launch_d<48>(op, s);
    case 64: return launch_d<64>(op, s);
    case 96: return launch_d<96>(op, s);
    case 128: return launch_d<128>(op, s);
    case 192: return launch_d<192>(op, s);          // cfg4 (bair_big, n_head_channels = 192): key tile 32
    case 256: return launch_d<256>(op, s);          // cfg7 (Cityscapes SPADE, n_head_channels = 256): one stage
    case 288: return launch_d<288>(op, s);          // cfg6 (UCF-101, n_head_channels = 288): one stage, split P V
    default: break;
  }
  set_error("ATTENTION_UMMA: head dim %d unsupported (32/48/64/96/128/192/256/288)", op.i1);
  return -1;
}

}  // namespace mcvd

extern "C" long long mcvd_attention_scratch_bytes(int B, int T, int C) {
  return mcvd::attention_umma_scratch_bytes(B, T, C);
}
