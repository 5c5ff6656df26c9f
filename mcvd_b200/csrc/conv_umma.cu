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
// Half mode (MCVD_F_HALF, template HALF): one product  hi*hi  per (tap, k16 step), the 11-bit significand of the
// TF32 convolutions cuDNN runs for the reference.  Only hi is converted and staged (a slab stage is one half image)
// and only hi is packed and streamed (a weight k16 step is 32 * NT bytes); everything else -- norm / FiLM / SiLU,
// raw TMA stages, work organisation, the epilogue -- is the same code.
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
// Warp roles (128 * (NWG + 1) threads, one CTA per SM, persistent over MT x NT tiles, MT = 64 * NWG positions):
//   warps 0-2   producers: raw fp32 NHWC stage in smem -> normalise/FiLM/SiLU -> fp16 hi/lo -> smem slab (2-3 stages)
//               (generic-proxy stores + fence.proxy.async).  Thread 0 also issues the TMA (cp.async.bulk.tensor)
//               loads of the raw input boxes and norm-table rows, one K-block ahead of the conversion.
//   warp  3     weight loader: cp.async.bulk (TMA 1-D) of pre-packed fp16 hi/lo smem images (ring of NB stages)
//   warps 4-    NWG = 2 or 3 consumer warpgroups, 64 rows of the tile each: wgmma m64nNTk16 from the slab and weight
//               stages, then the epilogue straight from the accumulator registers (bias / residual / scale /
//               SiLU, optional GroupNorm statistics of the stored output)
// Tile height.  The weight bytes streamed per MMA and the halo positions converted per output position both fall
// as 1/MT, so streaming convs with NT <= 192 run three consumer warpgroups (MT = 192): warpgroup 0 gives registers
// back (setmaxnreg) so that the consumers hold 96 accumulators each.  Statistics-writing and input-stationary
// launches keep MT = 128 (their statistics layout and slab stages are sized in 128-position tiles).  Every output
// sums the same products in the same order at either height, so the two give identical bits.
//
// Raw input stages.  The real pixels among consecutive padded-flat positions are consecutive NHWC pixels, so the
// raw input of a slab is one run of rows of a 2-D {C_src, B*H*W} tensor map: one TMA box of HP rows (two when
// HP > 256, the box-size limit), zero-filled past the end of the batch.  One-tap K-blocks (1x1 convs, the fused
// shortcut segment) load and convert only the MT rows of the tile's own positions.  The boxes are 64- / 128-byte
// swizzled (KB = 16 / 32 channels per row) so that eight producers reading the same 16 bytes of eight consecutive
// rows hit distinct banks.
#include <cuda.h>
#include <cuda_fp16.h>

#include <algorithm>
#include <cstring>

#include "mcvd_common.cuh"
#include "umma_ptx.cuh"

namespace mcvd {

constexpr int STAT_MT = 128;    // positions per tile of the statistics layout (the two-warpgroup tile)

namespace {

using namespace ptx;

constexpr int NPROD = 96;       // producer threads (warps 0-2)
constexpr int W_LOAD = 3;       // weight-loader warp
constexpr int W_CONS = 4;       // first consumer warp (warpgroups 1..NWG)
// NWG = 2: 384 threads, 168 registers each: room for the 128 accumulators of NT = 256.  NWG = 3: 512 threads launched
// at 128 registers; warpgroup 0 drops to 96 and the consumers rise to 136 (128 * 96 + 384 * 136 <= 65536), enough
// for the 96 accumulators of NT = 192 without spills (the producers spill below 88)
constexpr int NT_MAX3 = 192;
constexpr int REG_PROD3 = 96, REG_CONS3 = 136;
constexpr float STAT_SCALE = 65536.0f;   // fixed-point scale of the epilogue statistics
constexpr int TAB_NB = 8;       // images whose norm-table rows are staged in smem per K-block
constexpr int HP_MAX = 512;     // >= 192 + 2 * 130 rounded to 8 = 456, the MT = 192 slab at 128x128
constexpr int PPT = (HP_MAX + NPROD - 1) / NPROD;   // slab positions per producer thread
constexpr int RAW_STAGES = 2;   // raw input stages: the loads of K-block g + 1 fly while K-block g is converted
constexpr int MAX_RESIDENT = 12;   // K-blocks an input-stationary work item keeps resident (12 x 16 KB at KB = 32)

// tiled tensor maps of the raw sources s0..s3 ({C_src, B*H*W}) and of the norm table; unused entries are zero
struct ConvMaps {
  CUtensorMap src[4];
  CUtensorMap tab;
};

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
  int Qtot;              // total flat positions
  int KB;                // channels per K-block (16|32)
  int HP;                // halo slab positions (multiple of 8)
  int boxn, nbox;        // rows per TMA box of the first segment's sources, boxes per K-block
  int raw_off, raw_stage, tab_off;   // smem offset and size of a raw stage; its norm-table rows follow the pixels
  int RA;                // raw stages: RAW_STAGES, or 1 where two do not fit (the loads then wait for the conversion)
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
__device__ __forceinline__ int decode_pos(const ConvArgs& a, int q, int& b_out) {
  if (q < 0 || q >= a.Qtot) return -1;
  const int b = q / a.Pimg;
  const int r = q - b * a.Pimg;
  const int rr = r / a.Wp, cc = r - rr * a.Wp;
  b_out = b;
  if (a.ks == 3) {
    if (rr == 0 || cc == 0) return -1;
    return (b * a.H + (rr - 1)) * a.W + (cc - 1);
  }
  return (b * a.H + rr) * a.W + cc;
}

// first pixel index at or after flat position q (B*H*W past the end): the first row of a raw TMA box
__device__ __forceinline__ int first_raw(const ConvArgs& a, int q) {
  q = max(q, 0);
  if (q >= a.Qtot) return a.B * a.H * a.W;
  if (a.ks == 1) return q;
  const int b = q / a.Pimg;
  const int r = q - b * a.Pimg;
  const int rr = r / a.Wp, cc = r - rr * a.Wp;
  if (rr == 0) return b * a.H * a.W;
  return (b * a.H + (rr - 1)) * a.W + (cc == 0 ? 0 : cc - 1);
}

template <int NT, int NWG, bool HALF>
__global__ void __launch_bounds__(128 * (NWG + 1), 1) k_conv_umma(const ConvArgs a,
                                                                  const __grid_constant__ ConvMaps maps) {
  static_assert(NWG == 2 || (NWG == 3 && NT <= NT_MAX3), "three consumer warpgroups hold at most 96 accumulators");
  constexpr int MT = 64 * NWG;                                       // positions per tile
  constexpr int NTHREADS = 128 * (NWG + 1);
  constexpr int NCONS = 4 * NWG;                                     // consumer warps
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  const int chunks = a.KB / 8;
  const uint32_t a_half_bytes = (uint32_t)chunks * a.HP * 16;       // one of hi / lo
  const uint32_t a_stage_bytes = HALF ? a_half_bytes : 2 * a_half_bytes;
  constexpr uint32_t b_step_bytes = (HALF ? 32u : 64u) * NT;         // one k16 step: hi (2 chunks) [+ lo]
  const uint32_t b_stage_bytes = (uint32_t)(a.KB / 16) * b_step_bytes;
  uint8_t* a_base = smem_raw;
  uint8_t* b_base = a_base + (size_t)a.SA * a_stage_bytes;
  uint8_t* raw_base = smem_raw + a.raw_off;                          // [RA][raw_stage], 1024-byte aligned
  int* pinfo = reinterpret_cast<int*>(raw_base + (size_t)a.RA * a.raw_stage);   // [PPT][NPROD]
  unsigned long long* stat_s = reinterpret_cast<unsigned long long*>(pinfo + PPT * NPROD);   // [NJ][2][NT]
  uint64_t* bars = reinterpret_cast<uint64_t*>(stat_s + (a.stats ? a.NJ * 2 * NT : 0));
  // bars: a_full[SA], a_empty[SA], b_full[NB], b_empty[NB], r_full[RA]
  const uint32_t bar0 = smem_u32(bars);
  auto A_FULL = [&](int i) { return bar0 + 8u * i; };
  auto A_EMPTY = [&](int i) { return bar0 + 8u * (a.SA + i); };
  auto B_FULL = [&](int i) { return bar0 + 8u * (2 * a.SA + i); };
  auto B_EMPTY = [&](int i) { return bar0 + 8u * (2 * a.SA + a.NB + i); };
  auto R_FULL = [&](int i) { return bar0 + 8u * (2 * a.SA + 2 * a.NB + i); };
  const int groups_n = a.tiles_n / a.NPI;                 // work item t: m tile t / groups_n, n tiles of group t % groups_n

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int taps = a.ks * a.ks;

  if (tid == 0) {
    // consumers release a stage with one arrival per consumer warp
    for (int i = 0; i < a.SA; ++i) { mbar_init(A_FULL(i), NPROD); mbar_init(A_EMPTY(i), NCONS); }
    for (int i = 0; i < a.NB; ++i) { mbar_init(B_FULL(i), 1); mbar_init(B_EMPTY(i), NCONS); }
    for (int i = 0; i < a.RA; ++i) mbar_init(R_FULL(i), 1);
    fence_barrier_init();
  }
  if (a.stats)
    for (int i = tid; i < a.NJ * 2 * NT; i += NTHREADS) stat_s[i] = 0ull;
  __syncthreads();

  if (warp < W_CONS) {
    // warpgroup 0 (producers and weight loader) hands registers to the consumers; the branch structure lets ptxas
    // allocate each role within its budget
    if constexpr (NWG == 3) setmaxnreg_dec<REG_PROD3>();
    if (warp < W_LOAD) {
      // =========================== producers ===========================
      // One thread = one 8-channel chunk ch of the K-block over the slab positions h = h_lo + pp + k * ppass, so the
      // norm-table row of the current image stays in its registers.  Lane l of a warp takes chunk (l / 8) % chunks
      // and 32 / chunks consecutive positions per pass, so the eight threads of each quarter-warp read the same 16
      // bytes of eight consecutive raw rows (distinct banks under the swizzle) and store 128 contiguous bytes.  The
      // raw input and the (mean, rstd*G, S) rows of the <= tab_nb images the tile touches arrive by TMA in raw stage
      // g % RA.
      const bool has_tab = a.tab != nullptr;
      const int ch = (lane >> 3) % chunks;
      const int ppass = NPROD / chunks;                      // positions per pass: 24 (KB = 32) or 48 (KB = 16)
      const int pp = warp * (32 / chunks) + (lane & 7) + 8 * ((lane >> 3) / chunks);
      const uint32_t rowb = (uint32_t)a.KB * 4, smask = a.KB == 32 ? 7u : 3u;   // raw row bytes, swizzle row mask
      auto tile_b0_of = [&](int t) {
        const int q_first = (t / groups_n) * MT - a.halo0;
        return q_first <= 0 ? 0 : min(a.B - 1, q_first / a.Pimg);
      };
      // TMA issue (thread 0): K-block ikb of work item it, the ig-th K-block of this CTA
      const uint32_t raw0 = smem_u32(raw_base);
      const uint32_t main_bytes = (uint32_t)a.nbox * a.boxn * rowb, ctr_bytes = (uint32_t)MT * rowb;
      const uint32_t tab_bytes = (uint32_t)a.tab_nb * a.KB * (a.tab_planar ? 12 : 16);
      int it = blockIdx.x, ikb = 0, ig = 0;
      auto issue_next = [&]() {
        if (it >= a.ntiles) return;
        const int p0 = (it / groups_n) * MT;
        const bool seg2 = ikb >= a.nKB0;
        int si, cc0;
        if (!seg2) {
          const int c0 = ikb * a.KB;
          if (c0 < a.C0) { si = 0; cc0 = c0; } else { si = 1; cc0 = c0 - a.C0; }
        } else {
          const int c0 = (ikb - a.nKB0) * a.KB;
          if (c0 < a.C2) { si = 2; cc0 = c0; } else { si = 3; cc0 = c0 - a.C2; }
        }
        const bool use_tab = has_tab && !seg2;
        const uint32_t dst = raw0 + (uint32_t)(ig % a.RA) * a.raw_stage;
        const uint32_t bar = R_FULL(ig % a.RA);
        mbar_arrive_expect_tx(bar, (seg2 ? ctr_bytes : main_bytes) + (use_tab ? tab_bytes : 0u));
        if (seg2) {
          tma_load_2d(dst, &maps.src[si], cc0, first_raw(a, p0), bar);
        } else {
          const int r0 = first_raw(a, p0 - a.halo0);
          for (int i = 0; i < a.nbox; ++i)
            tma_load_2d(dst + (uint32_t)i * a.boxn * rowb, &maps.src[si], cc0, r0 + i * a.boxn, bar);
        }
        if (use_tab) {
          if (a.tab_planar) tma_load_3d(dst + a.tab_off, &maps.tab, ikb * a.KB, 0, tile_b0_of(it), bar);
          else tma_load_2d(dst + a.tab_off, &maps.tab, 4 * ikb * a.KB, tile_b0_of(it), bar);
        }
        ++ig;
        if (++ikb == a.nKB) { ikb = 0; it += gridDim.x; }
      };
      if (tid == 0)
        for (int i = 0; i < a.RA - 1; ++i) issue_next();
      int g = 0;                                             // K-blocks produced so far (all tiles)
      for (int t = blockIdx.x; t < a.ntiles; t += gridDim.x) {
        const int p0 = (t / groups_n) * MT;
        const int tb0 = tile_b0_of(t);
        // per tile, not per K-block: image slot << 16 | row in the first segment's raw box, or -1 for zero padding,
        // of each slab position.  Other producers read the entries (after the barrier at the top of the K-block
        // loop), so wait until all of them are done with the previous tile's.
        const int raw_m = first_raw(a, p0 - a.halo0), raw_c = first_raw(a, p0);
        named_bar_sync(1, NPROD);
        for (int h = tid; h < a.HP; h += NPROD) {
          int b = tb0;
          const int pix = decode_pos(a, p0 - a.halo0 + h, b);
          pinfo[h] = pix < 0 ? -1 : ((b - tb0) << 16) | (pix - raw_m);
        }
        for (int kb = 0; kb < a.nKB; ++kb, ++g) {
          const int st = g % a.SA;
          const bool seg2 = kb >= a.nKB0;
          const bool use_tab = has_tab && !seg2;
          // the second segment is read at the centre tap only: stage just the tile's own positions, from a box that
          // starts at the tile's first pixel
          const int h_lo = seg2 ? a.halo0 : 0, h_hi = seg2 ? a.halo0 + MT : a.HP;
          const int roff = seg2 ? raw_c - raw_m : 0;
          // every producer finished reading the raw stage of K-block g - 1: refill it with K-block g + RA - 1
          named_bar_sync(1, NPROD);
          if (tid == 0) issue_next();
          mbar_wait(A_EMPTY(st), ((g / a.SA) & 1) ^ 1);
          const int rs = g % a.RA;
          mbar_wait(R_FULL(rs), (g / a.RA) & 1);
          const uint8_t* raw = raw_base + (size_t)rs * a.raw_stage;
          const float* tsm = reinterpret_cast<const float*>(raw + a.tab_off);
          uint8_t* hi_base = a_base + (size_t)st * a_stage_bytes + (size_t)ch * a.HP * 16;
          uint8_t* lo_base = hi_base + a_half_bytes;
          // the 8 raw channels of chunk ch at slab position h (zeros at padding)
          auto load_raw = [&](int info, float4& r0, float4& r1) {
            r0 = r1 = make_float4(0.f, 0.f, 0.f, 0.f);
            if (info >= 0) {
              const uint32_t off = (uint32_t)((info & 0xffff) - roff) * rowb + 32u * ch;
              const uint32_t sw = ((off >> 7) & smask) << 4;
              r0 = *reinterpret_cast<const float4*>(raw + (off ^ sw));
              r1 = *reinterpret_cast<const float4*>(raw + ((off + 16u) ^ sw));
            }
          };
          // (mean, rstd*G, S) of the cached image's 8 channels; rstd*G is the same fp32 product for every position
          float tmean[8], tmul[8], tadd[8];
          int tcur = -1;
          int h = h_lo + pp;
          int info_n = h < h_hi ? pinfo[h] : -1;
          float4 n0, n1;
          load_raw(info_n, n0, n1);
#pragma unroll 1
          for (; h < h_hi; h += ppass) {
            const int info = info_n;
            const float4 c0 = n0, c1 = n1;
            // the next position's raw loads fly while this one is converted
            info_n = h + ppass < h_hi ? pinfo[h + ppass] : -1;
            load_raw(info_n, n0, n1);
            uint4 hv = make_uint4(0u, 0u, 0u, 0u), lv = hv;
            if (info >= 0) {
              float v[8] = {c0.x, c0.y, c0.z, c0.w, c1.x, c1.y, c1.z, c1.w};
              if (use_tab) {
                const int bidx = info >> 16;
                if (bidx != tcur) {
                  tcur = bidx;
                  if (a.tab_planar) {                        // [tab_nb][mean | rstd*G | S][KB]
                    const float* tb = tsm + bidx * 3 * a.KB + ch * 8;
#pragma unroll
                    for (int e = 0; e < 8; ++e) { tmean[e] = tb[e]; tmul[e] = tb[a.KB + e]; tadd[e] = tb[2 * a.KB + e]; }
                  } else {                                   // [tab_nb][KB] float4 (mean, rstd, G, S)
                    const float4* tb = reinterpret_cast<const float4*>(tsm) + bidx * a.KB + ch * 8;
#pragma unroll
                    for (int e = 0; e < 8; ++e) {
                      const float4 tv = tb[e];
                      tmean[e] = tv.x; tmul[e] = tv.y * tv.z; tadd[e] = tv.w;
                    }
                  }
                }
#pragma unroll
                for (int e = 0; e < 8; ++e) v[e] = fmaf(v[e] - tmean[e], tmul[e], tadd[e]);
                if (a.act_in) silu_fast8(v);
              }
              uint32_t hw[4], lw[4];
              if constexpr (HALF) {
#pragma unroll
                for (int e = 0; e < 4; ++e) hw[e] = cvt_hi2(v[2 * e], v[2 * e + 1]);
              } else {
#pragma unroll
                for (int e = 0; e < 4; ++e) split2(v[2 * e], v[2 * e + 1], hw[e], lw[e]);
                lv = make_uint4(lw[0], lw[1], lw[2], lw[3]);
              }
              hv = make_uint4(hw[0], hw[1], hw[2], hw[3]);
            }
            *reinterpret_cast<uint4*>(hi_base + (size_t)h * 16) = hv;
            if constexpr (!HALF) *reinterpret_cast<uint4*>(lo_base + (size_t)h * 16) = lv;
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
    }
  } else {
    if constexpr (NWG == 3) setmaxnreg_inc<REG_CONS3>();
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
      const int p0 = (t / groups_n) * MT;
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
            const uint64_t dah = desc_add(a_proto, a_tap16 + (uint32_t)(2 * s) * a_lbo16);
            wgmma_ss<NT>(acc, dah, dbh, 1);
            if constexpr (!HALF) {
              const uint64_t dbl = desc_add(dbh, b_lo16);
              const uint64_t dal = desc_add(dah, a_half16);
              if (a.split & 1) wgmma_ss<NT>(acc, dal, dbh, 1);
              if (a.split & 2) wgmma_ss<NT>(acc, dah, dbl, 1);
            }
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
      const int tile_b0 = min(a.B - 1, p0 / a.Pimg);
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
        // all warpgroups' sums of this tile -> global [tile][NJ][2][Cout]; re-zero for the next tile
        named_bar_sync(2, 32 * NCONS);
        const int et = tid - W_CONS * 32;
        unsigned long long* gp = a.stats + (size_t)(p0 / MT) * a.NJ * 2 * a.Cout;
        for (int i = et; i < a.NJ * 2 * NT; i += 32 * NCONS) {
          const int jp = i / NT, n = i - jp * NT;
          gp[(size_t)jp * a.Cout + n0 + n] = stat_s[i];
          stat_s[i] = 0ull;
        }
        named_bar_sync(2, 32 * NCONS);
      }
    }
  }
}

// ---- weight packing ---------------------------------------------------------------------------------
// in : w_taps fp32 [taps][Cin][Cout]
// out: fp16 stages of (KB/16) k16 steps, each  hi[2 chunks][NT][8]  then (parts = 2)  lo[2 chunks][NT][8]; stage of
//      (n tile nt, K-block kb, tap) = nt * per_unit + stage_off + kb * taps + tap.  parts = 1 is the half-mode image:
//      the same hi values, half the bytes.
__global__ void k_pack_weights(const float* __restrict__ w, __half* __restrict__ out, int taps, int Cin, int Cout,
                               int NT, int KB, float scale, int stage_off, int per_unit, int parts) {
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
    long long base = step * (2LL * parts * NT * 8);      // halfs per step: hi 2*NT*8 [+ lo 2*NT*8]
    long long o = (long long)(j * NT + n) * 8 + e;
    out[base + o] = h;
    if (parts == 2) out[base + 2LL * NT * 8 + o] = l;
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
  int boxn, nbox, tab_nb;   // first-segment TMA boxes; images whose norm-table rows a raw stage holds
  int raw_off, raw_stage, tab_off, RA;
  size_t smem;
};

constexpr size_t SMEM_LIMIT = 227 * 1024;

size_t round1024(size_t x) { return (x + 1023) & ~(size_t)1023; }

// shared-memory plan of one conv with MT-position tiles and SA slab stages (two raw stages where they fit); false
// when it does not fit.  vbytes = staged bytes per operand value: 4 (fp16 hi + lo) or 2 (half mode, hi only).
// Layout: slab stages, weight stages, raw stages (1024-byte aligned for the swizzled TMA boxes), position table,
// statistics, barriers.
bool make_plan(int H, int W, int ks, int KB, int NT, bool stats, int SA, int MT, int vbytes, Plan& p) {
  const int Wp = ks == 3 ? W + 1 : W;
  const int Pimg = ks == 3 ? (H + 1) * (W + 1) : H * W;
  const int halo0 = ks == 3 ? Wp + 1 : 0;
  p.HP = (MT + 2 * halo0 + 7) & ~7;
  p.NJ = (MT - 1) / Pimg + 2;
  if (p.HP > HP_MAX) return false;
  p.nbox = p.HP > 256 ? 2 : 1;                               // TMA boxes hold <= 256 rows
  p.boxn = p.nbox == 1 ? p.HP : ((p.HP / 2 + 7) & ~7);      // a multiple of 8 rows keeps box 2 swizzle-aligned
  p.tab_nb = std::min(p.HP / Pimg + 2, TAB_NB);
  p.tab_off = p.nbox * p.boxn * KB * 4;
  p.raw_stage = (int)round1024((size_t)p.tab_off + (size_t)p.tab_nb * KB * 16);
  const size_t a_stage = (size_t)(KB / 8) * p.HP * 8 * vbytes;
  const size_t b_stage = (size_t)(KB / 16) * 16 * vbytes * NT;
  const size_t stat_bytes = stats ? (size_t)p.NJ * 2 * NT * 8 : 0;
  const size_t pinfo_bytes = (size_t)PPT * NPROD * 4;
  size_t bar_bytes = 0, fixed = 0;
  for (p.RA = RAW_STAGES; p.RA >= 1; --p.RA) {
    bar_bytes = 8 * (2 * SA + 20 + p.RA);
    fixed = round1024(SA * a_stage) + (size_t)p.RA * p.raw_stage + pinfo_bytes + stat_bytes + bar_bytes;
    if (fixed + 2 * b_stage <= SMEM_LIMIT) break;
  }
  if (p.RA == 0) return false;
  p.NB = (int)((SMEM_LIMIT - fixed) / b_stage);
  if (p.NB > 10) p.NB = 10;
  p.raw_off = (int)round1024(SA * a_stage + (size_t)p.NB * b_stage);
  p.smem = (size_t)p.raw_off + (size_t)p.RA * p.raw_stage + pinfo_bytes + stat_bytes + bar_bytes;
  return p.smem <= SMEM_LIMIT;
}

using EncodeTiled = CUresult (*)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                 const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                 CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// cuTensorMapEncodeTiled from the driver the runtime already loaded (the library does not link libcuda)
EncodeTiled encode_tiled() {
  static const EncodeTiled fn = [] {
    void* f = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &q) != cudaSuccess ||
        q != cudaDriverEntryPointSuccess)
      f = nullptr;
    return reinterpret_cast<EncodeTiled>(f);
  }();
  return fn;
}

// tiled map of an fp32 tensor (dims innermost first, byte strides of dims 1..rank-1); zero fill out of range
int encode_map(CUtensorMap* m, const float* base, int rank, const cuuint64_t* dims, const cuuint64_t* strides,
               const cuuint32_t* box, CUtensorMapSwizzle swz, const char* name) {
  MCVD_CHECK(((uintptr_t)base & 15) == 0, "%s: TMA source %p is not 16-byte aligned", name, (const void*)base);
  for (int i = 0; i < rank; ++i)
    MCVD_CHECK(box[i] >= 1 && box[i] <= 256, "%s: TMA box dimension %u outside [1, 256]", name, box[i]);
  for (int i = 0; i < rank - 1; ++i)
    MCVD_CHECK(strides[i] % 16 == 0, "%s: TMA stride %llu bytes is not a multiple of 16", name,
               (unsigned long long)strides[i]);
  const EncodeTiled enc = encode_tiled();
  MCVD_CHECK(enc != nullptr, "%s: cuTensorMapEncodeTiled unavailable", name);
  const cuuint32_t estr[3] = {1, 1, 1};
  const CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, (cuuint32_t)rank, const_cast<float*>(base), dims, strides,
                         box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swz, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  MCVD_CHECK(r == CUDA_SUCCESS, "%s: cuTensorMapEncodeTiled failed (%d)", name, (int)r);
  return 0;
}

template <int NT, int NWG, bool HALF>
int launch_nt(const ConvArgs& a, const ConvMaps& m, size_t smem, int grid, cudaStream_t s) {
  cudaError_t e =
      cudaFuncSetAttribute(k_conv_umma<NT, NWG, HALF>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  MCVD_CHECK(e == cudaSuccess, "CONV_UMMA: cudaFuncSetAttribute failed: %s", cudaGetErrorString(e));
  k_conv_umma<NT, NWG, HALF><<<grid, 128 * (NWG + 1), smem, s>>>(a, m);
  MCVD_CUDA_LAUNCH_CHECK("conv_umma");
  return 0;
}

template <int NT, bool HALF>
int launch_nt(const ConvArgs& a, const ConvMaps& m, size_t smem, int grid, int nwg, cudaStream_t s) {
  if constexpr (NT <= NT_MAX3)
    if (nwg == 3) return launch_nt<NT, 3, HALF>(a, m, smem, grid, s);
  return launch_nt<NT, 2, HALF>(a, m, smem, grid, s);
}

template <int NT>
int launch_nt(const ConvArgs& a, const ConvMaps& m, size_t smem, int grid, int nwg, bool half, cudaStream_t s) {
  return half ? launch_nt<NT, true>(a, m, smem, grid, nwg, s) : launch_nt<NT, false>(a, m, smem, grid, nwg, s);
}

// Launch plan of one conv on `sms` SMs: the kernel arguments, the shared-memory plan, the tile height and the grid.
// Host arithmetic only; launch_conv runs exactly this plan.  planar = the CONV_UMMA2 variant (planar norm table,
// K-block fixed by the caller when i2 != 0, statistics tiles padded to pairs).
int plan_conv(const McvdOp& op, int sms, bool planar, ConvArgs& a, Plan& p, int& MT, int& grid) {
  const char* name = planar ? "CONV_UMMA2" : "CONV_UMMA";
  MCVD_CHECK(op.src0 && op.w && op.dst && (op.C1 == 0 || op.src1), "%s: null pointer", name);
  MCVD_CHECK(op.i0 == 1 || op.i0 == 3, "%s: kernel size %d unsupported", name, op.i0);
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
  const bool half = (op.flags & MCVD_F_HALF) != 0;
  MCVD_CHECK(!half || op.i3 == 0 || op.i3 == 3, "%s: operand split %d with MCVD_F_HALF (one product; 0 or 3)", name,
             op.i3);
  const int vbytes = half ? 2 : 4;
  if (a.ks == 3) { a.Wp = op.W + 1; a.Pimg = (op.H + 1) * (op.W + 1); }
  else { a.Wp = op.W; a.Pimg = op.H * op.W; }
  MCVD_CHECK((long long)op.B * a.Pimg < (1LL << 31), "%s: too many pixels", name);
  a.Qtot = op.B * a.Pimg;
  MCVD_CHECK(!a.stats || a.Pimg >= 64, "%s: epilogue statistics need images of >= 64 positions", name);
  a.halo0 = (a.ks == 3) ? a.Wp + 1 : 0;
  a.nKB0 = (op.C0 + op.C1) / a.KB;
  a.nKB = a.nKB0 + (a.C2 + a.C3) / a.KB;
  a.tiles_n = op.Cout / NT;
  const long long tiles128 = (a.Qtot + STAT_MT - 1) / STAT_MT;
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
  const bool can_stay = a.ks == 1 && a.nKB == a.nKB0 && a.tiles_n > 1 && a.nKB <= MAX_RESIDENT &&
                        make_plan(op.H, op.W, a.ks, a.KB, NT, a.stats != nullptr, a.nKB, STAT_MT, vbytes, p);
  const bool stay = can_stay && (mode == 2 || (mode == 0 && 2 * tiles128 >= sms));
  // Slab stages of a streaming conv (CONV_UMMA i5, diagnostics): 0 = the launcher's choice, 2 or 3 forces them.
  const int sa_req = planar ? 0 : op.i5;
  MCVD_CHECK(sa_req == 0 || ((sa_req == 2 || sa_req == 3) && !stay), "%s: %d slab stages", name, sa_req);
  a.SA = stay ? a.nKB : (sa_req ? sa_req : 2);
  a.NPI = stay ? a.tiles_n : 1;
  // Tile height (CONV_UMMA i4, diagnostics): 0 = 192 positions (three consumer warpgroups) for a streaming conv
  // without statistics whose n tile fits the accumulator registers and whose plan fits shared memory with at least
  // three weight stages, unless it leaves the last SMs with more positions to cover (ceil(items / SMs) * MT): at 8x8
  // the 192-position items are too few to cover the SMs.  Measured on an H100 80GB HBM3 (700 W), MT = 128 -> 192:
  // with two weight stages (64x64 at NT = 192, next to the larger slab and raw stages) the weight ring stalls the
  // MMAs, 64x64 192->192 827 -> 1280 us; the 64x64 3x3 convs without a second segment, whose slab is 1.71x the tile,
  // gain from the smaller share of halo positions now that the producers keep up: 288->96 862 -> 758 us, 192->96
  // 612 -> 521 us.  128 or 192 forces the height (an error where 192 cannot run).
  // A third slab stage (i5 = 3) lets the producers run two K-blocks ahead, but it costs weight stages: at 64x64 it
  // measured 192->96 608 -> 581 us at MT = 128, 521 -> 535 us at MT = 192 and 859 -> 1331 us for 192->192 at
  // MT = 128, so the launcher keeps two.
  const int mt_req = planar ? 0 : op.i4;
  MCVD_CHECK(mt_req == 0 || mt_req == 128 || mt_req == 192, "%s: tile height %d", name, mt_req);
  const bool can3 = !planar && NT <= NT_MAX3 && !stay && !a.stats &&
                    make_plan(op.H, op.W, a.ks, a.KB, NT, false, a.SA, 192, vbytes, p) &&
                    (!a.tab || p.HP / a.Pimg + 2 <= TAB_NB);
  MCVD_CHECK(mt_req != 192 || can3, "%s: 192-position tiles need streaming, NT <= %d, no statistics and %dx%d to fit",
             name, NT_MAX3, op.H, op.W);
  auto last_positions = [&](int mt) {
    const long long items = (a.Qtot + mt - 1) / mt * a.tiles_n;
    return (items + sms - 1) / sms * mt;
  };
  MT = mt_req ? mt_req : (can3 && p.NB >= 3 && last_positions(192) <= last_positions(128) ? 192 : 128);
  long long tiles_m = (a.Qtot + MT - 1) / MT;
  if (planar) tiles_m = (tiles_m + 1) & ~1LL;          // the statistics array is sized in tile pairs: write all of it
  MCVD_CHECK(make_plan(op.H, op.W, a.ks, a.KB, NT, a.stats != nullptr, a.SA, MT, vbytes, p),
             "%s: tile does not fit shared memory (W=%d)", name, op.W);
  a.HP = p.HP; a.NB = p.NB; a.NJ = p.NJ;
  a.boxn = p.boxn; a.nbox = p.nbox; a.raw_off = p.raw_off; a.raw_stage = p.raw_stage; a.tab_off = p.tab_off;
  a.RA = p.RA;
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
  grid = a.ntiles < sms ? a.ntiles : sms;
  return 0;
}

int launch_conv(const McvdOp& op, cudaStream_t s, bool planar) {
  const char* name = planar ? "CONV_UMMA2" : "CONV_UMMA";
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  ConvArgs a;
  Plan p;
  int MT = 0, grid = 0;
  if (plan_conv(op, sms, planar, a, p, MT, grid)) return -1;
  const int NT = op.i1;
  const bool half = (op.flags & MCVD_F_HALF) != 0;
  // TMA maps: sources as {C, B*H*W} rows of KB channels, swizzled; the norm table as {4*Cin, B} or {Cin, 3, B}
  ConvMaps maps;
  memset(&maps, 0, sizeof(maps));
  {
    const float* srcs[4] = {a.s0, a.s1, a.s2, a.s3};
    const int cs[4] = {a.C0, a.C1, a.C2, a.C3};
    const CUtensorMapSwizzle swz = a.KB == 32 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B;
    for (int i = 0; i < 4; ++i) {
      if (!cs[i]) continue;
      MCVD_CHECK(srcs[i] != nullptr, "%s: null source %d", name, i);
      const cuuint64_t dims[2] = {(cuuint64_t)cs[i], (cuuint64_t)op.B * op.H * op.W};
      const cuuint64_t strides[1] = {(cuuint64_t)cs[i] * 4};
      const cuuint32_t box[2] = {(cuuint32_t)a.KB, (cuuint32_t)(i < 2 ? a.boxn : MT)};
      if (encode_map(&maps.src[i], srcs[i], 2, dims, strides, box, swz, name)) return -1;
    }
    if (a.tab) {
      const int Cin = op.C0 + op.C1;
      if (planar) {
        const cuuint64_t dims[3] = {(cuuint64_t)Cin, 3, (cuuint64_t)op.B};
        const cuuint64_t strides[2] = {(cuuint64_t)Cin * 4, (cuuint64_t)Cin * 12};
        const cuuint32_t box[3] = {(cuuint32_t)a.KB, 3, (cuuint32_t)a.tab_nb};
        if (encode_map(&maps.tab, a.tab, 3, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_NONE, name)) return -1;
      } else {
        const cuuint64_t dims[2] = {(cuuint64_t)Cin * 4, (cuuint64_t)op.B};
        const cuuint64_t strides[1] = {(cuuint64_t)Cin * 16};
        const cuuint32_t box[2] = {(cuuint32_t)(4 * a.KB), (cuuint32_t)a.tab_nb};
        if (encode_map(&maps.tab, a.tab, 2, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_NONE, name)) return -1;
      }
    }
  }
  switch (NT) {
#define MCVD_NT_CASE(n) case n: return launch_nt<n>(a, maps, p.smem, grid, MT / 64, half, s);
    MCVD_NT_CASE(16) MCVD_NT_CASE(32) MCVD_NT_CASE(48) MCVD_NT_CASE(64) MCVD_NT_CASE(80) MCVD_NT_CASE(96)
    MCVD_NT_CASE(112) MCVD_NT_CASE(128) MCVD_NT_CASE(144) MCVD_NT_CASE(160) MCVD_NT_CASE(176) MCVD_NT_CASE(192)
    MCVD_NT_CASE(208) MCVD_NT_CASE(224) MCVD_NT_CASE(240) MCVD_NT_CASE(256)
#undef MCVD_NT_CASE
    default: break;
  }
  MCVD_CHECK(false, "%s: n tile %d", name, NT);
}

long long pack(const float* w_taps, int taps, int Cin, int Cout, int n_tile, int KB, void* out, int scale_log2,
               int stage_off, int per_unit, int parts, void* stream) {
  if ((KB != 16 && KB != 32) || Cin % KB || n_tile < 16 || n_tile % 16 || Cout % n_tile) {
    set_error("umma_pack_weights: Cin %d / Cout %d / n_tile %d / KB %d unsupported", Cin, Cout, n_tile, KB);
    return -1;
  }
  if (parts != 1 && parts != 2) {
    set_error("umma_pack_weights: parts %d (1 = hi, 2 = hi + lo)", parts);
    return -1;
  }
  const long long bytes = (long long)taps * Cin * Cout * 2 * parts;      // fp16 hi [+ lo]
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
                                                                      scale, stage_off, per_unit, parts);
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

extern "C" int mcvd_conv_umma_launch_info(const McvdOp* op, int sms, int* out) {
  if (!op || !out || sms < 1 || (op->kind != MCVD_OP_CONV_UMMA && op->kind != MCVD_OP_CONV_UMMA2)) {
    mcvd::set_error("conv_umma_launch_info: needs a CONV_UMMA or CONV_UMMA2 op, an output array and sms >= 1");
    return -1;
  }
  mcvd::ConvArgs a;
  mcvd::Plan p;
  int MT = 0, grid = 0;
  if (mcvd::plan_conv(*op, sms, op->kind == MCVD_OP_CONV_UMMA2, a, p, MT, grid)) return -1;
  out[0] = a.KB; out[1] = MT; out[2] = a.SA; out[3] = a.NB; out[4] = a.RA; out[5] = a.NPI; out[6] = a.ntiles;
  out[7] = grid; out[8] = (int)p.smem;
  return 0;
}

extern "C" int mcvd_umma_kblock(int C0, int C1) { return mcvd::pick_kb(C0, C1); }

extern "C" long long mcvd_umma_pack_weights(const float* w_taps, int taps, int Cin, int Cout, int n_tile, int KB,
                                            void* out, int scale_log2, void* stream) {
  return mcvd::pack(w_taps, taps, Cin, Cout, n_tile, KB, out, scale_log2, 0, KB ? (Cin / KB) * taps : 0, 2, stream);
}

extern "C" long long mcvd_umma_pack_weights_ex(const float* w_taps, int taps, int Cin, int Cout, int n_tile, int KB,
                                               void* out, int scale_log2, int stage_off, int per_unit, int parts,
                                               void* stream) {
  return mcvd::pack(w_taps, taps, Cin, Cout, n_tile, KB, out, scale_log2, stage_off, per_unit, parts, stream);
}

extern "C" int mcvd_umma2_plan(int H, int W, int ks, int C0, int C1, int C2, int C3, int n_tile, int stats) {
  const int kb = mcvd::conv_kb(C0, C1, C2, C3);
  mcvd::Plan p;
  if (!kb || n_tile < 16 || n_tile > 256 || n_tile % 16) return 0;
  return mcvd::make_plan(H, W, ks, kb, n_tile, stats != 0, 2, mcvd::STAT_MT, 4, p) ? kb : 0;
}

// shared-memory plan of a conv (diagnostics / tests): out[0..9] = KB, HP, image stages, raw-input stages, weight
// stages, image slots per tile, accumulator columns outside registers (0), dynamic shared memory bytes, tiles
// per unit (1), accumulator sets (1); returns 0, or -1
extern "C" int mcvd_umma2_plan_info(int H, int W, int ks, int C0, int C1, int C2, int C3, int n_tile, int stats,
                                    int* out) {
  const int kb = mcvd_umma2_plan(H, W, ks, C0, C1, C2, C3, n_tile, stats);
  if (!kb || !out) return -1;
  mcvd::Plan p;
  mcvd::make_plan(H, W, ks, kb, n_tile, stats != 0, 2, mcvd::STAT_MT, 4, p);
  out[0] = kb; out[1] = p.HP; out[2] = 2; out[3] = p.RA; out[4] = p.NB; out[5] = p.NJ; out[6] = 0;
  out[7] = (int)p.smem; out[8] = 1; out[9] = 1;
  return 0;
}

extern "C" long long mcvd_umma2_stats_bytes(int B, int H, int W, int ks, int Cout) {
  const long long pimg = ks == 3 ? (long long)(H + 1) * (W + 1) : (long long)H * W;
  const long long tiles = 2 * ((B * pimg + 2 * mcvd::STAT_MT - 1) / (2 * mcvd::STAT_MT));
  const long long nj = (mcvd::STAT_MT - 1) / pimg + 2;
  return tiles * nj * 2 * Cout * 8;
}

extern "C" long long mcvd_umma2_pack_weights(const float* w_taps, int taps, int Cin, int Cout, int n_tile, int KB,
                                             void* out, int scale_log2, int stage_off, int per_unit, void* stream) {
  return mcvd::pack(w_taps, taps, Cin, Cout, n_tile, KB, out, scale_log2, stage_off, per_unit, 2, stream);
}
