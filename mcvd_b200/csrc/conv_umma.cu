// 3x3 (pad 1) / 1x1 convolution on the Hopper tensor cores (wgmma, fp32 accumulators in registers), with the
// GroupNorm / FiLM / SiLU input transform fused into the shared-memory staging.  Serves MCVD_OP_CONV_UMMA and
// MCVD_OP_CONV_UMMA2 (same kernel; the second reads the planar norm table and always pads the tile count to pairs).
//
// Reference semantics: nn.Conv2d 3x3 / 1x1 and NIN of models/better/layers.py:89-113,541-544 applied
// to get_act_norm's output (layerspp.py:518-549), i.e. Conv_0 / Conv_1 / Conv_2 / NIN_* of
// ResnetBlockBigGANppGN (layerspp.py:595-624) and AttnBlockpp (:230-249).
//
// fp32 parity on fp16 tensor cores: both operands are split  v = hi + lo  (hi = fp16(v),
// lo = fp16(v - hi)) and three MMAs  hi*hi + lo*hi + hi*lo  accumulate in fp32; the dropped
// lo*lo term and the second-level rounding are ~2^-22 relative.  Weights are pre-scaled by a power of
// two (undone in the epilogue) so their lo parts stay in the fp16 normal range.
//
// "Padded-flat" implicit GEMM.  The batch is viewed as one flat array of positions
//     q = b*(H+1)*(W+1) + r*(W+1) + c,   r in [0,H], c in [0,W],   pixel (y,x) = (r-1, c-1)
// where row r = 0 and column c = 0 are zero padding shared between neighbouring rows / images.  In
// this indexing every 3x3 tap is a CONSTANT flat offset  dy*(W+1) + dx,  so a CTA stages ONE halo
// slab [tile + 2*(W+1) + 2 positions] x [KB channels] of the transformed input in shared memory per
// K-block and all nine taps are shifted views of it: the A-operand descriptor of tap (dy,dx) is the
// slab descriptor advanced by (dy*(W+1)+dx) * 16 bytes.  That needs a layout whose M-stride is 16
// bytes, which is exactly the canonical no-swizzle K-major core-matrix layout
//     [k-chunk of 8 halfs][position][8 halfs = 16 B]      LBO = positions*16 B,  SBO = 128 B.
// Outputs at padding positions are computed and discarded (2..20 % of the rows).
//
// Warp roles (384 threads, one CTA per SM, persistent over 128-position x NT tiles):
//   warps 0-2   producers: fp32 NHWC global -> normalise/FiLM/SiLU -> fp16 hi/lo -> smem slab (2 stages)
//               (generic-proxy stores + fence.proxy.async)
//   warp  3     weight loader: cp.async.bulk (TMA 1-D) of pre-packed fp16 hi/lo smem images (ring of NB stages)
//   warps 4-11  two consumer warpgroups, 64 rows of the tile each: wgmma m64nNTk16 from the slab and weight
//               stages, then the epilogue straight from the accumulator registers (bias / residual / scale /
//               SiLU, optional GroupNorm statistics of the stored output)
#include <cuda_fp16.h>

#include "mcvd_common.cuh"
#include "umma_ptx.cuh"

namespace mcvd {

constexpr int MT = 128;         // positions per tile (two consumer warpgroups x 64)

namespace {

using namespace ptx;

constexpr int NPROD = 96;       // producer threads (warps 0-2)
constexpr int W_LOAD = 3;       // weight-loader warp
constexpr int W_CONS = 4;       // first consumer warp (warpgroups 1 and 2)
constexpr int NTHREADS = 384;   // 168 registers per thread: room for the 128 accumulators of NT = 256
constexpr float STAT_SCALE = 65536.0f;   // fixed-point scale of the epilogue statistics
constexpr int TAB_NB = 8;       // images whose norm-table rows are staged in smem per K-block
constexpr int HP_MAX = 512;
constexpr int MAX_RESIDENT = 12;   // K-blocks an input-stationary work item keeps resident (12 x 8 KB at KB = 32)

struct ConvArgs {
  const float* s0;
  const float* s1;
  const float* s2;       // second K-segment (fused 1x1 shortcut): raw sources, centre tap only
  const float* s3;
  int C2, C3, nKB0;      // nKB0 = K-blocks of the first segment; K-blocks >= nKB0 belong to the second
  const __half* wpk;     // packed weights (see k_pack_weights)
  const float* bias;
  const float* res;
  const float* tab;      // norm table or null: [B][Cin] float4 (mean, rstd, G, S), or planar [B][3][Cin]
  int tab_planar;        //   (mean | rstd*G | S) when tab_planar
  float* dst;
  unsigned long long* stats;   // optional: [tiles128][NJ][2][Cout] fixed-point sum / sum of squares of the stored output
  int NJ;                // image slots per 128-position tile (127 / Pimg + 2)
  int B, H, W, C0, C1, Cout;
  int ks;                // 1 or 3
  int Wp, Pimg;          // padded row pitch, positions per image
  long long Qtot;        // total flat positions
  int KB;                // channels per K-block (16|32)
  int HP;                // halo slab positions (multiple of 8)
  int halo0;             // slab index of the tile's first output position
  int nKB;               // K-blocks
  int NB;                // weight ring stages
  int SA;                // slab stages: 2 (streaming), or nKB (input-stationary: the m tile's whole input resident)
  int NPI;               // n tiles per work item: 1 (streaming) or tiles_n (input-stationary)
  int tiles_n, ntiles;   // n tiles per m tile, work items
  int act_in, act_out;
  int split;             // operand split (accuracy experiments): bit 0 = lo*hi term, bit 1 = hi*lo term
  int tab_nb;            // images a tile's slab can touch
  float wscale, oscale;
};

// position decode: flat q -> pixel index (b*H + y)*W + x, or -1 for padding / out of range
__device__ __forceinline__ int decode_pos(const ConvArgs& a, long long q, int& b_out) {
  if (q < 0 || q >= a.Qtot) return -1;
  const int b = (int)(q / a.Pimg);
  const int r = (int)(q - (long long)b * a.Pimg);
  const int rr = r / a.Wp, cc = r - rr * a.Wp;
  b_out = b;
  if (a.ks == 3) {
    if (rr == 0 || cc == 0) return -1;
    return (b * a.H + (rr - 1)) * a.W + (cc - 1);
  }
  return (b * a.H + rr) * a.W + cc;
}

template <int NT>
__global__ void __launch_bounds__(NTHREADS, 1) k_conv_umma(const ConvArgs a) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  const int chunks = a.KB / 8;
  const uint32_t a_half_bytes = (uint32_t)chunks * a.HP * 16;       // one of hi / lo
  const uint32_t a_stage_bytes = 2 * a_half_bytes;
  constexpr uint32_t b_step_bytes = 64u * NT;                        // one k16 step: hi (2 chunks) + lo
  const uint32_t b_stage_bytes = (uint32_t)(a.KB / 16) * b_step_bytes;
  uint8_t* a_base = smem_raw;
  uint8_t* b_base = a_base + (size_t)a.SA * a_stage_bytes;
  float* tab_s = reinterpret_cast<float*>(b_base + (size_t)a.NB * b_stage_bytes);         // [2][TAB_NB][96]
  unsigned long long* stat_s = reinterpret_cast<unsigned long long*>(tab_s + 2 * TAB_NB * 96);   // [NJ][2][NT]
  uint64_t* bars = reinterpret_cast<uint64_t*>(stat_s + (a.stats ? a.NJ * 2 * NT : 0));
  // bars: a_full[SA], a_empty[SA], b_full[NB], b_empty[NB]
  const uint32_t bar0 = smem_u32(bars);
  auto A_FULL = [&](int i) { return bar0 + 8u * i; };
  auto A_EMPTY = [&](int i) { return bar0 + 8u * (a.SA + i); };
  auto B_FULL = [&](int i) { return bar0 + 8u * (2 * a.SA + i); };
  auto B_EMPTY = [&](int i) { return bar0 + 8u * (2 * a.SA + a.NB + i); };
  const int groups_n = a.tiles_n / a.NPI;                 // work item t: m tile t / groups_n, n tiles of group t % groups_n

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int taps = a.ks * a.ks;

  if (tid == 0) {
    // consumers release a stage with one arrival per consumer warp (8)
    for (int i = 0; i < a.SA; ++i) { mbar_init(A_FULL(i), NPROD); mbar_init(A_EMPTY(i), 8); }
    for (int i = 0; i < a.NB; ++i) { mbar_init(B_FULL(i), 1); mbar_init(B_EMPTY(i), 8); }
    fence_barrier_init();
  }
  if (a.stats)
    for (int i = tid; i < a.NJ * 2 * NT; i += NTHREADS) stat_s[i] = 0ull;
  __syncthreads();

  if (warp < W_LOAD) {
    // =========================== producers ===========================
    // One thread = one slab position x all KB channels of the K-block at a time; the (mean, rstd*G, S) rows of the
    // <= TAB_NB images the tile touches are staged in smem per K-block (double-buffered, one barrier per K-block).
    const int Cin = a.C0 + a.C1;
    const bool has_tab = a.tab != nullptr;
    auto tile_b0_of = [&](int t) {
      const long long q_first = (long long)(t / groups_n) * MT - a.halo0;
      return q_first <= 0 ? 0 : (int)min((long long)(a.B - 1), q_first / a.Pimg);
    };
    int g = 0;                                             // K-blocks produced so far (all tiles)
    for (int t = blockIdx.x; t < a.ntiles; t += gridDim.x) {
      const long long p0 = (long long)(t / groups_n) * MT;
      const int tb0 = tile_b0_of(t);
      for (int kb = 0; kb < a.nKB; ++kb, ++g) {
        const int st = g % a.SA;
        const float* src; int cs, cc0;
        const bool seg2 = kb >= a.nKB0;
        if (!seg2) {
          const int c0 = kb * a.KB;
          if (c0 < a.C0) { src = a.s0; cs = a.C0; cc0 = c0; } else { src = a.s1; cs = a.C1; cc0 = c0 - a.C0; }
        } else {
          const int c0 = (kb - a.nKB0) * a.KB;
          if (c0 < a.C2) { src = a.s2; cs = a.C2; cc0 = c0; } else { src = a.s3; cs = a.C3; cc0 = c0 - a.C2; }
        }
        const bool use_tab = has_tab && !seg2;
        float* tsm = tab_s + (size_t)(g & 1) * TAB_NB * 96;
        if (use_tab) {
          for (int i = tid; i < a.tab_nb * a.KB; i += NPROD) {
            const int bi = i / a.KB, c = i - bi * a.KB;
            const int b = min(tb0 + bi, a.B - 1);
            const int ch = kb * a.KB + c;
            float m, gs, sh;
            if (a.tab_planar) {
              const float* tp = a.tab + (long long)b * 3 * Cin + ch;
              m = __ldg(tp); gs = __ldg(tp + Cin); sh = __ldg(tp + 2 * Cin);
            } else {
              const float4 tv = __ldg(reinterpret_cast<const float4*>(a.tab) + (long long)b * Cin + ch);
              m = tv.x; gs = tv.y * tv.z; sh = tv.w;
            }
            tsm[bi * 96 + c] = m; tsm[bi * 96 + 32 + c] = gs; tsm[bi * 96 + 64 + c] = sh;
          }
        }
        mbar_wait(A_EMPTY(st), ((g / a.SA) & 1) ^ 1);
        // this K-block's table is complete, and every producer finished reading the buffer written two K-blocks ago
        named_bar_sync(1, NPROD);
        uint8_t* hi_base = a_base + (size_t)st * a_stage_bytes;
        uint8_t* lo_base = hi_base + a_half_bytes;
#pragma unroll 1
        for (int h = tid; h < a.HP; h += NPROD) {
          int b = tb0;
          const int pix = decode_pos(a, p0 - a.halo0 + h, b);
          const int bidx = b - tb0;
          float4 raw[8];
#pragma unroll
          for (int j = 0; j < 8; ++j)
            if (j < 2 * chunks) raw[j] = pix >= 0 ? __ldg(reinterpret_cast<const float4*>(src + (long long)pix * cs + cc0) + j)
                                                  : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
          for (int ch = 0; ch < 4; ++ch) {
            if (ch < chunks) {
              uint4 hv = make_uint4(0u, 0u, 0u, 0u), lv = hv;
              if (pix >= 0) {
                float v[8] = {raw[2 * ch].x, raw[2 * ch].y, raw[2 * ch].z, raw[2 * ch].w,
                              raw[2 * ch + 1].x, raw[2 * ch + 1].y, raw[2 * ch + 1].z, raw[2 * ch + 1].w};
                if (use_tab) {
                  const float* tb = tsm + bidx * 96 + ch * 8;
#pragma unroll
                  for (int e = 0; e < 8; ++e) v[e] = fmaf(v[e] - tb[e], tb[32 + e], tb[64 + e]);
                  if (a.act_in) silu_fast8(v);
                }
                uint32_t hw[4], lw[4];
#pragma unroll
                for (int e = 0; e < 4; ++e) split2(v[2 * e], v[2 * e + 1], hw[e], lw[e]);
                hv = make_uint4(hw[0], hw[1], hw[2], hw[3]);
                lv = make_uint4(lw[0], lw[1], lw[2], lw[3]);
              }
              const size_t off = ((size_t)ch * a.HP + h) * 16;
              *reinterpret_cast<uint4*>(hi_base + off) = hv;
              *reinterpret_cast<uint4*>(lo_base + off) = lv;
            }
          }
        }
        fence_proxy_async();          // make the generic-proxy stores visible to the tensor-core (async) proxy
        mbar_arrive(A_FULL(st));
      }
    }
  } else if (warp == W_LOAD) {
    // =========================== weight loader ===========================
    if (elect_one()) {
      const uint32_t b0 = smem_u32(b_base);
      const int per_tile = a.nKB0 * taps + (a.nKB - a.nKB0);          // second segment: one (centre) tap per K-block
      int st = 0, ph = 1;
      for (int t = blockIdx.x; t < a.ntiles; t += gridDim.x)
       for (int j = 0; j < a.NPI; ++j) {
        const int nt = (t % groups_n) * a.NPI + j;
        const uint8_t* wsrc = reinterpret_cast<const uint8_t*>(a.wpk) + (size_t)nt * per_tile * b_stage_bytes;
        for (int i = 0; i < per_tile; ++i) {
          mbar_wait(B_EMPTY(st), ph);
          mbar_arrive_expect_tx(B_FULL(st), b_stage_bytes);
          bulk_g2s(b0 + (uint32_t)st * b_stage_bytes, wsrc + (size_t)i * b_stage_bytes, b_stage_bytes, B_FULL(st));
          if (++st == a.NB) { st = 0; ph ^= 1; }
        }
      }
    }
    __syncwarp();
  } else {
    // =========================== consumers (MMA + epilogue) ===========================
    const int wg = (warp - W_CONS) >> 2;                   // rows [64 wg, 64 wg + 64) of the tile
    const int wq = (warp - W_CONS) & 3;                             // warp within the warpgroup: rows 16 wq .. 16 wq + 15
    const int ksteps = a.KB / 16;
    const uint32_t a_lbo = (uint32_t)a.HP * 16;
    const uint64_t a_proto = make_desc(0, a_lbo, 128), b_proto = make_desc(0, NT * 16, 128);
    const uint32_t a_half16 = a_half_bytes >> 4, b_lo16 = 2u * NT;
    const uint32_t a0_16 = smem_u32(a_base) >> 4, b0_16 = smem_u32(b_base) >> 4;
    const uint32_t a_stage16 = a_stage_bytes >> 4, b_stage16 = b_stage_bytes >> 4;
    const uint32_t a_lbo16 = a_lbo >> 4;
    int bst = 0, bph = 0, g0 = 0;                          // g0: first K-block (all items) of the current item
    for (int t = blockIdx.x; t < a.ntiles; t += gridDim.x, g0 += a.nKB)
     for (int j = 0; j < a.NPI; ++j) {
      const long long p0 = (long long)(t / groups_n) * MT;
      const int n0 = ((t % groups_n) * a.NPI + j) * NT;
      const bool last_n = j == a.NPI - 1;                  // the slab stages are released after the item's last n tile
      float acc[NT / 2];
#pragma unroll
      for (int i = 0; i < NT / 2; ++i) acc[i] = 0.f;
      // the stage whose wgmmas were committed last and not yet released (one group stays in flight)
      int pend_b = -1, pend_a = -1;
      for (int kb = 0; kb < a.nKB; ++kb) {
        const int g = g0 + kb;
        const int st = g % a.SA;
        mbar_wait(A_FULL(st), (g / a.SA) & 1);
        const uint32_t a_hi16 = a0_16 + (uint32_t)st * a_stage16 + (uint32_t)(a.halo0 + 64 * wg);
        const int ntap = (kb < a.nKB0) ? taps : 1;
        for (int tap = 0; tap < ntap; ++tap) {
          mbar_wait(B_FULL(bst), bph);
          const int shift = (a.ks == 3 && kb < a.nKB0) ? ((tap / 3 - 1) * a.Wp + (tap % 3 - 1)) : 0;
          const uint32_t a_tap16 = a_hi16 + (uint32_t)shift;
          const uint32_t b_tap16 = b0_16 + (uint32_t)bst * b_stage16;
          wgmma_fence();
#pragma unroll 1
          for (int s = 0; s < ksteps; ++s) {
            const uint64_t dbh = desc_add(b_proto, b_tap16 + (uint32_t)s * (b_step_bytes >> 4));
            const uint64_t dbl = desc_add(dbh, b_lo16);
            const uint64_t dah = desc_add(a_proto, a_tap16 + (uint32_t)(2 * s) * a_lbo16);
            const uint64_t dal = desc_add(dah, a_half16);
            wgmma_ss<NT>(acc, dah, dbh, 1);
            if (a.split & 1) wgmma_ss<NT>(acc, dal, dbh, 1);
            if (a.split & 2) wgmma_ss<NT>(acc, dah, dbl, 1);
          }
          wgmma_commit();
          wgmma_wait<1>();                                 // the previous group is complete: release its stages
          if (pend_b >= 0 && lane == 0) mbar_arrive(B_EMPTY(pend_b));
          if (pend_a >= 0 && lane == 0) mbar_arrive(A_EMPTY(pend_a));
          pend_b = bst;
          pend_a = (tap == ntap - 1 && last_n) ? st : -1;
          if (++bst == a.NB) { bst = 0; bph ^= 1; }
        }
      }
      wgmma_wait<0>();
#pragma unroll
      for (int i = 0; i < NT / 2; ++i) reg_fence(acc[i]);
      if (lane == 0) { mbar_arrive(B_EMPTY(pend_b)); if (pend_a >= 0) mbar_arrive(A_EMPTY(pend_a)); }

      // ---- epilogue: thread owns rows r and r + 8, two adjacent columns of every 8-column block ----
      const int r0 = 64 * wg + 16 * wq + (lane >> 2);
      const int cq = 2 * (lane & 3);
      int pix[2], slot[2];
      const int tile_b0 = (int)min((long long)(a.B - 1), p0 / a.Pimg);
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        int b = 0;
        pix[i] = decode_pos(a, p0 + r0 + 8 * i, b);
        slot[i] = pix[i] >= 0 ? b - tile_b0 : -1;
      }
      unsigned jmask = 0;
      if (a.stats) {
#pragma unroll 1
        for (int jj = 0; jj < a.NJ; ++jj)
          if (__ballot_sync(0xffffffffu, slot[0] == jj || slot[1] == jj)) jmask |= 1u << jj;
      }
#pragma unroll
      for (int j = 0; j < NT / 8; ++j) {
        const int n = n0 + 8 * j + cq;
        const float2 bv = a.bias ? __ldg(reinterpret_cast<const float2*>(a.bias + n)) : make_float2(0.f, 0.f);
        float v[2][2];
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          float2 rv = make_float2(0.f, 0.f);
          if (a.res && pix[i] >= 0) rv = __ldg(reinterpret_cast<const float2*>(a.res + (long long)pix[i] * a.Cout + n));
          float x0 = (acc[4 * j + 2 * i] * a.wscale + bv.x + rv.x) * a.oscale;     // wscale: power of two, exact
          float x1 = (acc[4 * j + 2 * i + 1] * a.wscale + bv.y + rv.y) * a.oscale;
          if (a.act_out) { x0 = silu_f(x0); x1 = silu_f(x1); }
          v[i][0] = x0; v[i][1] = x1;
          if (pix[i] >= 0) *reinterpret_cast<float2*>(a.dst + (long long)pix[i] * a.Cout + n) = make_float2(x0, x1);
        }
        if (a.stats) {
#pragma unroll 1
          for (int jj = 0; jj < a.NJ; ++jj) {
            if (!(jmask & (1u << jj))) continue;
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              long long s1 = 0;
              unsigned long long s2 = 0;
#pragma unroll
              for (int i = 0; i < 2; ++i) {
                if (slot[i] == jj) {
                  const int xi = __float2int_rn(v[i][e] * STAT_SCALE);          // saturates at +-2^31
                  s1 += xi;
                  s2 += (unsigned long long)((long long)xi * (long long)xi);
                }
              }
#pragma unroll
              for (int o = 4; o <= 16; o <<= 1) {
                s1 += __shfl_xor_sync(0xffffffffu, s1, o);
                s2 += __shfl_xor_sync(0xffffffffu, s2, o);
              }
              if (lane < 4) {
                unsigned long long* sp = stat_s + (size_t)jj * 2 * NT + 8 * j + cq + e;
                atomicAdd(sp, (unsigned long long)s1);
                atomicAdd(sp + NT, s2);
              }
            }
          }
        }
      }
      if (a.stats) {
        // both warpgroups' sums of this 128-position tile -> global [tile128][NJ][2][Cout]; re-zero for the next tile
        named_bar_sync(2, 256);
        const int et = tid - W_CONS * 32;
        unsigned long long* gp = a.stats + (size_t)(p0 / MT) * a.NJ * 2 * a.Cout;
        for (int i = et; i < a.NJ * 2 * NT; i += 256) {
          const int jp = i / NT, n = i - jp * NT;
          gp[(size_t)jp * a.Cout + n0 + n] = stat_s[i];
          stat_s[i] = 0ull;
        }
        named_bar_sync(2, 256);
      }
    }
  }
}

// ---- weight packing ---------------------------------------------------------------------------------
// in : w_taps fp32 [taps][Cin][Cout]
// out: fp16 stages of (KB/16) k16 steps, each  hi[2 chunks][NT][8]  then  lo[2 chunks][NT][8]; stage of
//      (n tile nt, K-block kb, tap) = nt * per_unit + stage_off + kb * taps + tap
__global__ void k_pack_weights(const float* __restrict__ w, __half* __restrict__ out, int taps, int Cin, int Cout,
                               int NT, int KB, float scale, int stage_off, int per_unit) {
  const int ksteps = KB / 16, nKB = Cin / KB, nNT = Cout / NT;
  const long long total = (long long)nNT * nKB * taps * ksteps * 2 * NT * 8;  // (chunk j, n, e) per step
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    int e = (int)(i % 8);
    long long t = i / 8;
    int n = (int)(t % NT); t /= NT;
    int j = (int)(t % 2); t /= 2;
    int s = (int)(t % ksteps); t /= ksteps;
    int tap = (int)(t % taps); t /= taps;
    int kb = (int)(t % nKB); t /= nKB;
    int nt = (int)t;
    int c = kb * KB + s * 16 + j * 8 + e;
    float v = w[((long long)tap * Cin + c) * Cout + nt * NT + n] * scale;
    __half h = __float2half_rn(v);
    __half l = __float2half_rn(v - __half2float(h));
    long long step = ((long long)nt * per_unit + stage_off + (long long)kb * taps + tap) * ksteps + s;
    long long base = step * (4LL * NT * 8);      // halfs per step: hi 2*NT*8 + lo 2*NT*8
    long long o = (long long)(j * NT + n) * 8 + e;
    out[base + o] = h;
    out[base + 2LL * NT * 8 + o] = l;
  }
}

int pick_kb(int C0, int C1) {
  if (C0 % 32 == 0 && C1 % 32 == 0) return 32;
  if (C0 % 16 == 0 && C1 % 16 == 0) return 16;
  return 0;
}

// K-block of a conv with a (C0|C1) main source and an optional (C2|C3) shortcut segment; 0 = not runnable
int conv_kb(int C0, int C1, int C2, int C3) {
  int kb = pick_kb(C0, C1);
  if (C2 + C3 > 0 && pick_kb(C2, C3) < kb) kb = pick_kb(C2, C3);
  return kb;
}

struct Plan {
  int HP, NB, NJ;
  size_t smem;
};

constexpr size_t SMEM_LIMIT = 227 * 1024;

// shared-memory plan of one conv with SA slab stages; false when it does not fit
bool make_plan(int H, int W, int ks, int KB, int NT, bool stats, int SA, Plan& p) {
  const int Wp = ks == 3 ? W + 1 : W;
  const int Pimg = ks == 3 ? (H + 1) * (W + 1) : H * W;
  const int halo0 = ks == 3 ? Wp + 1 : 0;
  p.HP = (MT + 2 * halo0 + 7) & ~7;
  p.NJ = (MT - 1) / Pimg + 2;
  if (p.HP > HP_MAX) return false;
  const size_t a_stage = (size_t)2 * (KB / 8) * p.HP * 16;
  const size_t b_stage = (size_t)(KB / 16) * 64 * NT;
  const size_t stat_bytes = stats ? (size_t)p.NJ * 2 * NT * 8 : 0;
  const size_t fixed = SA * a_stage + (size_t)2 * TAB_NB * 96 * 4 + stat_bytes + 8 * (2 * SA + 20);   // ... + barriers
  if (fixed + 2 * b_stage > SMEM_LIMIT) return false;
  p.NB = (int)((SMEM_LIMIT - fixed) / b_stage);
  if (p.NB > 10) p.NB = 10;
  p.smem = fixed + (size_t)p.NB * b_stage;
  return true;
}

template <int NT>
int launch_nt(const ConvArgs& a, size_t smem, int grid, cudaStream_t s) {
  cudaError_t e = cudaFuncSetAttribute(k_conv_umma<NT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  MCVD_CHECK(e == cudaSuccess, "CONV_UMMA: cudaFuncSetAttribute failed: %s", cudaGetErrorString(e));
  k_conv_umma<NT><<<grid, NTHREADS, smem, s>>>(a);
  MCVD_CUDA_LAUNCH_CHECK("conv_umma");
  return 0;
}

// common launcher: planar = the CONV_UMMA2 variant (planar norm table, K-block fixed by the caller when i2 != 0,
// statistics tiles padded to pairs)
int launch_conv(const McvdOp& op, cudaStream_t s, bool planar) {
  const char* name = planar ? "CONV_UMMA2" : "CONV_UMMA";
  MCVD_CHECK(op.src0 && op.w && op.dst && (op.C1 == 0 || op.src1), "%s: null pointer", name);
  MCVD_CHECK(op.i0 == 1 || op.i0 == 3, "%s: kernel size %d unsupported", name, op.i0);
  ConvArgs a;
  a.s0 = (const float*)op.src0; a.s1 = (const float*)op.src1; a.wpk = (const __half*)op.w;
  a.s2 = (const float*)op.src2; a.s3 = (const float*)op.src3; a.C2 = op.src2 ? op.C2 : 0; a.C3 = op.src3 ? op.C3 : 0;
  a.bias = (const float*)op.bias; a.res = (const float*)op.aux0; a.tab = (const float*)op.aux1;
  a.tab_planar = planar ? 1 : 0;
  a.dst = (float*)op.dst;
  a.stats = (unsigned long long*)op.dst2;
  a.B = op.B; a.H = op.H; a.W = op.W; a.C0 = op.C0; a.C1 = op.C1; a.Cout = op.Cout; a.ks = op.i0;
  const int NT = op.i1;
  a.KB = conv_kb(op.C0, op.C1, a.C2, a.C3);
  MCVD_CHECK(a.KB != 0, "%s: input channels (%d,%d | %d,%d) must be multiples of 16", name, op.C0, op.C1, a.C2, a.C3);
  MCVD_CHECK(!planar || op.i2 == 0 || op.i2 == a.KB, "CONV_UMMA2: weights packed for K-block %d, the conv uses %d",
             op.i2, a.KB);
  MCVD_CHECK(NT >= 16 && NT <= 256 && NT % 16 == 0 && op.Cout % NT == 0, "%s: n tile %d invalid for Cout %d", name, NT,
             op.Cout);
  if (a.ks == 3) { a.Wp = op.W + 1; a.Pimg = (op.H + 1) * (op.W + 1); }
  else { a.Wp = op.W; a.Pimg = op.H * op.W; }
  a.Qtot = (long long)op.B * a.Pimg;
  MCVD_CHECK((long long)op.B * op.H * op.W < (1LL << 31) && a.Qtot < (1LL << 31), "%s: too many pixels", name);
  MCVD_CHECK(!a.stats || a.Pimg >= 64, "%s: epilogue statistics need images of >= 64 positions", name);
  a.halo0 = (a.ks == 3) ? a.Wp + 1 : 0;
  a.nKB0 = (op.C0 + op.C1) / a.KB;
  a.nKB = a.nKB0 + (a.C2 + a.C3) / a.KB;
  a.tiles_n = op.Cout / NT;
  long long tiles_m = (a.Qtot + MT - 1) / MT;
  if (planar) tiles_m = (tiles_m + 1) & ~1LL;          // the statistics array is sized in tile pairs: write all of it
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  // Work organisation (CONV_UMMA i2): 1 = streaming, one (m tile, n tile) per work item through two slab stages;
  // 2 = input-stationary, one m tile per work item with its whole input resident (one slab stage per K-block) while
  // the weights of every n tile stream past it, so the input is read and transformed once instead of once per n
  // tile (1x1 convs without a second segment, <= MAX_RESIDENT K-blocks; otherwise streaming).  0 = input-stationary
  // where it applies and there are at least half as many m tiles as SMs, else streaming.  Measured per 1x1 conv of
  // cfg2 (B = 64) on an H100 80GB HBM3 (700 W), streaming -> input-stationary: 32x32 192->576 359 -> 260 us,
  // 16x16 288->864 231 -> 130 us (128 m tiles), 8x8 288->288 37 -> 49 us (32 m tiles: too few work items).
  // tools/time_conv1x1.py repeats the measurement.
  const int mode = planar ? 0 : op.i2;
  MCVD_CHECK(mode >= 0 && mode <= 2, "%s: work organisation %d", name, mode);
  Plan p;
  const bool can_stay = a.ks == 1 && a.nKB == a.nKB0 && a.tiles_n > 1 && a.nKB <= MAX_RESIDENT &&
                        make_plan(op.H, op.W, a.ks, a.KB, NT, a.stats != nullptr, a.nKB, p);
  const bool stay = can_stay && (mode == 2 || (mode == 0 && 2 * tiles_m >= sms));
  a.SA = stay ? a.nKB : 2;
  a.NPI = stay ? a.tiles_n : 1;
  MCVD_CHECK(make_plan(op.H, op.W, a.ks, a.KB, NT, a.stats != nullptr, a.SA, p),
             "%s: tile does not fit shared memory (W=%d)", name, op.W);
  a.HP = p.HP; a.NB = p.NB; a.NJ = p.NJ;
  a.act_in = (op.flags & MCVD_F_ACT_IN) ? 1 : 0;
  a.act_out = (op.flags & MCVD_F_ACT_OUT) ? 1 : 0;
  a.wscale = op.f1; a.oscale = op.f0;
  a.split = (op.i3 >= 1 && op.i3 <= 3) ? op.i3 : (op.i3 == 4 ? 0 : 3);
  {
    const int nb = a.HP / a.Pimg + 2;
    MCVD_CHECK(nb <= TAB_NB || !a.tab, "%s: %dx%d images are too small for the fused-norm path", name, op.H, op.W);
    a.tab_nb = (nb <= TAB_NB) ? nb : 0;
  }
  MCVD_CHECK(tiles_m * a.tiles_n < (1LL << 31), "%s: too many tiles", name);
  a.ntiles = (int)(tiles_m * (a.tiles_n / a.NPI));
  const int grid = a.ntiles < sms ? a.ntiles : sms;
  switch (NT) {
#define MCVD_NT_CASE(n) case n: return launch_nt<n>(a, p.smem, grid, s);
    MCVD_NT_CASE(16) MCVD_NT_CASE(32) MCVD_NT_CASE(48) MCVD_NT_CASE(64) MCVD_NT_CASE(80) MCVD_NT_CASE(96)
    MCVD_NT_CASE(112) MCVD_NT_CASE(128) MCVD_NT_CASE(144) MCVD_NT_CASE(160) MCVD_NT_CASE(176) MCVD_NT_CASE(192)
    MCVD_NT_CASE(208) MCVD_NT_CASE(224) MCVD_NT_CASE(240) MCVD_NT_CASE(256)
#undef MCVD_NT_CASE
    default: break;
  }
  MCVD_CHECK(false, "%s: n tile %d", name, NT);
}

long long pack(const float* w_taps, int taps, int Cin, int Cout, int n_tile, int KB, void* out, int scale_log2,
               int stage_off, int per_unit, void* stream) {
  if ((KB != 16 && KB != 32) || Cin % KB || n_tile < 16 || n_tile % 16 || Cout % n_tile) {
    set_error("umma_pack_weights: Cin %d / Cout %d / n_tile %d / KB %d unsupported", Cin, Cout, n_tile, KB);
    return -1;
  }
  const long long bytes = (long long)taps * Cin * Cout * 4;      // hi + lo fp16
  if (!out) return bytes;
  if (!w_taps) {
    set_error("umma_pack_weights: null input");
    return -1;
  }
  const float scale = ldexpf(1.0f, scale_log2);
  const long long total = (long long)taps * Cin * Cout;
  long long blocks = (total + 255) / 256;
  if (blocks > 132LL * 16) blocks = 132LL * 16;
  k_pack_weights<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(w_taps, (__half*)out, taps, Cin, Cout, n_tile, KB,
                                                                      scale, stage_off, per_unit);
  if (cudaGetLastError() != cudaSuccess) {
    set_error("umma_pack_weights: launch failed");
    return -2;
  }
  return bytes;
}

}  // namespace

int launch_conv_umma(const McvdOp& op, cudaStream_t s) { return launch_conv(op, s, false); }
int launch_conv_umma2(const McvdOp& op, cudaStream_t s) { return launch_conv(op, s, true); }

}  // namespace mcvd

extern "C" int mcvd_umma_kblock(int C0, int C1) { return mcvd::pick_kb(C0, C1); }

extern "C" long long mcvd_umma_pack_weights(const float* w_taps, int taps, int Cin, int Cout, int n_tile, int KB,
                                            void* out, int scale_log2, void* stream) {
  return mcvd::pack(w_taps, taps, Cin, Cout, n_tile, KB, out, scale_log2, 0, KB ? (Cin / KB) * taps : 0, stream);
}

extern "C" int mcvd_umma2_plan(int H, int W, int ks, int C0, int C1, int C2, int C3, int n_tile, int stats) {
  const int kb = mcvd::conv_kb(C0, C1, C2, C3);
  mcvd::Plan p;
  if (!kb || n_tile < 16 || n_tile > 256 || n_tile % 16) return 0;
  return mcvd::make_plan(H, W, ks, kb, n_tile, stats != 0, 2, p) ? kb : 0;
}

// shared-memory plan of a conv (diagnostics / tests): out[0..9] = KB, HP, image stages, raw-ring stages (0), weight
// stages, image slots per tile, accumulator columns outside registers (0), dynamic shared memory bytes, tiles
// per unit (1), accumulator sets (1); returns 0, or -1
extern "C" int mcvd_umma2_plan_info(int H, int W, int ks, int C0, int C1, int C2, int C3, int n_tile, int stats,
                                    int* out) {
  const int kb = mcvd_umma2_plan(H, W, ks, C0, C1, C2, C3, n_tile, stats);
  if (!kb || !out) return -1;
  mcvd::Plan p;
  mcvd::make_plan(H, W, ks, kb, n_tile, stats != 0, 2, p);
  out[0] = kb; out[1] = p.HP; out[2] = 2; out[3] = 0; out[4] = p.NB; out[5] = p.NJ; out[6] = 0;
  out[7] = (int)p.smem; out[8] = 1; out[9] = 1;
  return 0;
}

extern "C" long long mcvd_umma2_stats_bytes(int B, int H, int W, int ks, int Cout) {
  const long long pimg = ks == 3 ? (long long)(H + 1) * (W + 1) : (long long)H * W;
  const long long tiles = 2 * ((B * pimg + 2 * mcvd::MT - 1) / (2 * mcvd::MT));
  const long long nj = (mcvd::MT - 1) / pimg + 2;
  return tiles * nj * 2 * Cout * 8;
}

extern "C" long long mcvd_umma2_pack_weights(const float* w_taps, int taps, int Cin, int Cout, int n_tile, int KB,
                                             void* out, int scale_log2, int stage_off, int per_unit, void* stream) {
  return mcvd::pack(w_taps, taps, Cin, Cout, n_tile, KB, out, scale_log2, stage_off, per_unit, stream);
}
