// Multi-head self-attention over the H*W tokens of one sample (AttnBlockpp.forward,
// reference models/better/layerspp.py:239-245), flash-style: the [T, T] score matrix the reference
// materialises (4 MB per sample-head at 32x32) never leaves the SM.  fp32 FFMA, online softmax.
//
//   qkv [B, T, 3C] (q | k | v along channels, head h = channels [h*d, (h+1)*d)),  out [B, T, C]
//   grid = (T/64 query tiles, heads, B), 256 threads; key/value tiles of 64 tokens.
//   S tile 64x64: thread (ty,tx) owns rows 4ty..4ty+3, cols 4tx..4tx+3   (q, k kept k-major in smem)
//   O tile 64xd : thread (ty,tx) owns rows 4ty..4ty+3, cols {tx*V + 16*V*r + v}
#include "mcvd_common.cuh"

namespace mcvd {

namespace {

constexpr int TQ = 64, TK = 64, LDT = 68;  // k-major q/k tiles padded to 68 floats per row

template <int V, int NCH>
__global__ void __launch_bounds__(256) k_attention(const float* __restrict__ qkv, float* __restrict__ out, int T,
                                                   int C, int d, float scale) {
  extern __shared__ __align__(16) float smem[];
  float* Qt = smem;                 // [d][LDT]
  float* Kt = Qt + d * LDT;         // [d][LDT]
  float* Vs = Kt + d * LDT;         // [TK][d]
  float* Pt = Vs + TK * d;          // [TK][LDT]  (P transposed: Pt[j][i])

  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int q0 = blockIdx.x * TQ, h = blockIdx.y, b = blockIdx.z;
  const int C3 = 3 * C;
  const float* base = qkv + (long long)b * T * C3 + h * d;

  // Q tile -> Qt[c][i]  (lanes walk tokens => conflict-free transposed stores)
  for (int idx = tid; idx < TQ * (d / 4); idx += 256) {
    int i = idx & 63, c4 = idx >> 6;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (q0 + i < T) v = *reinterpret_cast<const float4*>(base + (long long)(q0 + i) * C3 + c4 * 4);
    Qt[(c4 * 4 + 0) * LDT + i] = v.x;
    Qt[(c4 * 4 + 1) * LDT + i] = v.y;
    Qt[(c4 * 4 + 2) * LDT + i] = v.z;
    Qt[(c4 * 4 + 3) * LDT + i] = v.w;
  }

  float o[4][NCH * V];
  float mrow[4], lrow[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    mrow[i] = -INFINITY;
    lrow[i] = 0.f;
#pragma unroll
    for (int j = 0; j < NCH * V; ++j) o[i][j] = 0.f;
  }

  for (int k0 = 0; k0 < T; k0 += TK) {
    __syncthreads();  // previous tile fully consumed (also orders the Q stores before first use)
    for (int idx = tid; idx < TK * (d / 4); idx += 256) {
      int j = idx & 63, c4 = idx >> 6;
      float4 kv = make_float4(0.f, 0.f, 0.f, 0.f), vv = kv;
      if (k0 + j < T) {
        const float* p = base + (long long)(k0 + j) * C3 + c4 * 4;
        kv = *reinterpret_cast<const float4*>(p + C);
        vv = *reinterpret_cast<const float4*>(p + 2 * C);
      }
      Kt[(c4 * 4 + 0) * LDT + j] = kv.x;
      Kt[(c4 * 4 + 1) * LDT + j] = kv.y;
      Kt[(c4 * 4 + 2) * LDT + j] = kv.z;
      Kt[(c4 * 4 + 3) * LDT + j] = kv.w;
      *reinterpret_cast<float4*>(&Vs[j * d + c4 * 4]) = vv;
    }
    __syncthreads();

    // S = Q K^T
    float sacc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) sacc[i][j] = 0.f;
    for (int c = 0; c < d; ++c) {
      float4 qv = *reinterpret_cast<const float4*>(&Qt[c * LDT + ty * 4]);
      float4 kv = *reinterpret_cast<const float4*>(&Kt[c * LDT + tx * 4]);
      float qa[4] = {qv.x, qv.y, qv.z, qv.w}, ka[4] = {kv.x, kv.y, kv.z, kv.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) sacc[i][j] = fmaf(qa[i], ka[j], sacc[i][j]);
    }

    // online softmax; the 16 threads sharing `ty` are a half-warp
    float corr[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float mx = -INFINITY;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        float sv = (k0 + tx * 4 + j < T) ? sacc[i][j] * scale : -INFINITY;
        sacc[i][j] = sv;
        mx = fmaxf(mx, sv);
      }
#pragma unroll
      for (int off = 8; off > 0; off >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, off));
      float mnew = fmaxf(mrow[i], mx);
      float sum = 0.f;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        float p = expf(sacc[i][j] - mnew);
        sacc[i][j] = p;
        sum += p;
      }
#pragma unroll
      for (int off = 8; off > 0; off >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, off);
      corr[i] = expf(mrow[i] - mnew);
      lrow[i] = lrow[i] * corr[i] + sum;
      mrow[i] = mnew;
    }
    // P -> smem transposed (Pt[j][i]); each thread writes its 4x4 block
#pragma unroll
    for (int j = 0; j < 4; ++j)
      *reinterpret_cast<float4*>(&Pt[(tx * 4 + j) * LDT + ty * 4]) =
          make_float4(sacc[0][j], sacc[1][j], sacc[2][j], sacc[3][j]);
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < NCH * V; ++j) o[i][j] *= corr[i];
    __syncthreads();

    // O += P V
    for (int j = 0; j < TK; ++j) {
      float4 pv = *reinterpret_cast<const float4*>(&Pt[j * LDT + ty * 4]);
      float pa[4] = {pv.x, pv.y, pv.z, pv.w};
#pragma unroll
      for (int r = 0; r < NCH; ++r) {
        float vv[V];
        const float* vp = &Vs[j * d + tx * V + 16 * V * r];
        if constexpr (V == 4) {
          float4 t = *reinterpret_cast<const float4*>(vp);
          vv[0] = t.x; vv[1] = t.y; vv[2] = t.z; vv[3] = t.w;
        } else if constexpr (V == 2) {
          float2 t = *reinterpret_cast<const float2*>(vp);
          vv[0] = t.x; vv[1] = t.y;
        } else {
          vv[0] = *vp;
        }
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int v = 0; v < V; ++v) o[i][r * V + v] = fmaf(pa[i], vv[v], o[i][r * V + v]);
      }
    }
  }

  // normalise and store
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    int t = q0 + ty * 4 + i;
    if (t >= T) continue;
    float inv = 1.0f / lrow[i];
    float* op = out + ((long long)b * T + t) * C + h * d;
#pragma unroll
    for (int r = 0; r < NCH; ++r)
#pragma unroll
      for (int v = 0; v < V; ++v) op[tx * V + 16 * V * r + v] = o[i][r * V + v] * inv;
  }
}

template <int V, int NCH>
int launch_one(const McvdOp& op, cudaStream_t s) {
  int T = op.H * op.W, d = op.i1, heads = op.i0;
  size_t smem = (size_t)(2 * d * LDT + TK * d + TK * LDT) * sizeof(float);
  // per-device attribute: set on every launch (cheap, legal during stream capture)
  cudaError_t e = cudaFuncSetAttribute(k_attention<V, NCH>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  MCVD_CHECK(e == cudaSuccess, "ATTENTION: cudaFuncSetAttribute(%zu B) failed: %s", smem, cudaGetErrorString(e));
  dim3 grid(cdiv(T, TQ), heads, op.B);
  k_attention<V, NCH><<<grid, 256, smem, s>>>((const float*)op.src0, (float*)op.dst, T, op.C0, d, op.f0);
  MCVD_CUDA_LAUNCH_CHECK("attention");
  return 0;
}

}  // namespace

// the head dims launch_attention runs; any T (the last key tile is partial)
int attention_simt_key_tile(int T, int d) {
  switch (d) {
    case 16: case 32: case 48: case 64: case 96: case 128: case 192: case 256: return T > 0 ? TK : 0;
    default: return 0;
  }
}

int launch_attention(const McvdOp& op, cudaStream_t s) {
  MCVD_CHECK(op.src0 && op.dst, "ATTENTION: null pointer");
  int d = op.i1, heads = op.i0;
  MCVD_CHECK(heads * d == op.C0, "ATTENTION: heads %d x dim %d != channels %d", heads, d, op.C0);
  switch (d) {
    case 16: return launch_one<1, 1>(op, s);
    case 32: return launch_one<2, 1>(op, s);
    case 48: return launch_one<1, 3>(op, s);
    case 64: return launch_one<4, 1>(op, s);
    case 96: return launch_one<2, 3>(op, s);
    case 128: return launch_one<4, 2>(op, s);
    case 192: return launch_one<4, 3>(op, s);
    case 256: return launch_one<4, 4>(op, s);
    default: break;
  }
  set_error("ATTENTION: head dim %d unsupported (16/32/48/64/96/128/192/256)", d);
  return -1;
}

}  // namespace mcvd
