// Geometry, validation and activation gather of the evaluation networks' convolutions and max-pools (LPIPS, I3D,
// Inception-v3): MCVD_OP_CONV_RELU, MCVD_OP_CONV3D, MCVD_OP_MAXPOOL3D, MCVD_OP_CONV2D, MCVD_OP_MAXPOOL2D and the
// _TF32 conv kinds.  The fp32 FFMA kernels (conv_eval.cu) and the TF32 tensor-core kernel (conv_tf32.cu) both gather
// through the functions here, so they read the same input values for every (position, k).
#pragma once

#include <math.h>

#include "mcvd_common.cuh"

namespace mcvd {

// Implicit-GEMM geometry: M = images * To * Ho * Wo output positions, N = Cout, K = kt * kh * kw * Cin in
// (dt, dy, dx, c) order.  The input is [images, Tin, Hin, Win, Cin] (a 2-D op has Tin = kt = To = 1).  Hc x Wc is
// the extent G_S2MAX's window moves over, the input's 3x3 / stride-2 max-pool (Hin x Win for the other modes).  Strides st (time) and ss (space), front pads pt, ph, pw.  The output is channels [off, off + Cout) of
// a pitch-wide map.  A max-pool uses the same fields with Cout = Cin and K unused.
struct ConvGeom {
  int Tin, Hin, Win, Cin, Hc, Wc;
  int kt, kh, kw, st, ss, pt, ph, pw;
  int To, Ho, Wo, Cout, K, pitch, off;
  long long M;
};

// Gather modes: how the activation of (position, k) is read.
//   G_CONV2 / G_CONV3: any 2-D / 3-D window, stride and padding (2-D keeps no time axis in its index arithmetic);
//   G_PW: 1x1(x1) stride 1, where the output position is the input position and k the channel;
//   G_BMAX / G_BAVG: G_PW over the 3x3 / stride-1 / pad-1 pool of the input (Inception's branch_pool convs): max,
//     where padding never wins, or the average with count_include_pad=False (the sum of the taps inside the map over
//     their number);
//   G_S2MAX: G_CONV2 over the 3x3 / stride-2 max-pool of the input (AlexNet features[2], [5]).
enum { G_CONV2 = 0, G_CONV3 = 1, G_PW = 2, G_BMAX = 3, G_BAVG = 4, G_S2MAX = 5 };

// NULL with g filled in, or why the op is unusable.  Covers every kind listed at the top; a _TF32 kind is checked as
// its fp32 kind.  Shared by validation and launch (conv_eval.cu).
const char* conv_geom(const McvdOp& op, ConvGeom& g);
// conv_geom, then the tile grid of the TF32 kernel (conv_tf32.cu)
const char* conv_tf32_geom(const McvdOp& op, ConvGeom& g);
// the gather mode of a conv op that conv_geom accepted
int gather_mode(const McvdOp& op);
// "CONV_RELU", "CONV3D", ... for messages
const char* conv_kind_name(int kind);

// the output position one loader thread gathers for, decomposed once per CTA (not once per K slice)
struct ConvPos {
  const float* img;          // the position's image / video (its input pixel for G_PW), NULL past the last position
  int it0, iy0, ix0;         // front-top-left input coordinate of its window (the position itself for the branch pools)
};

struct ConvTap {
  int c, dt, dy, dx;         // channel and window offsets of k (c = k for the modes without a window)
  bool in;                   // k < K
};

template <int MODE>
__device__ __forceinline__ ConvPos conv_pos(const float* __restrict__ src, const ConvGeom& g, long long m) {
  ConvPos q{nullptr, 0, 0, 0};
  if (m >= g.M) return q;
  if (MODE == G_PW) {
    q.img = src + m * g.Cin;
    return q;
  }
  const int hw = g.Ho * g.Wo;
  const int P = MODE == G_CONV3 ? g.To * hw : hw;
  const long long n = m / P;
  int r = (int)(m - n * P);
  if (MODE == G_CONV3) {
    const int ot = r / hw;
    r -= ot * hw;
    q.it0 = ot * g.st - g.pt;
    q.img = src + n * g.Tin * g.Hin * g.Win * g.Cin;
  } else {
    q.img = src + n * g.Hin * g.Win * g.Cin;
  }
  const int oy = r / g.Wo;
  q.iy0 = oy * g.ss - g.ph;
  q.ix0 = (r - oy * g.Wo) * g.ss - g.pw;
  return q;
}

template <int MODE>
__device__ __forceinline__ ConvTap conv_tap(const ConvGeom& g, int k) {
  ConvTap t{k, 0, 0, 0, k < g.K};
  if ((MODE != G_CONV2 && MODE != G_CONV3 && MODE != G_S2MAX) || !t.in) return t;
  const int tap = k / g.Cin;
  t.c = k - tap * g.Cin;
  int r = tap;
  if (MODE == G_CONV3) {
    const int khw = g.kh * g.kw;
    t.dt = tap / khw;
    r = tap - t.dt * khw;
  }
  t.dy = r / g.kw;
  t.dx = r - t.dy * g.kw;
  return t;
}

__device__ __forceinline__ float4 ld4(const float* p) { return *reinterpret_cast<const float4*>(p); }

__device__ __forceinline__ void max4(float4& v, const float4& u) {
  v.x = fmaxf(v.x, u.x); v.y = fmaxf(v.y, u.y); v.z = fmaxf(v.z, u.z); v.w = fmaxf(v.w, u.w);
}

// The 4 consecutive-k activations of (q, t): zero past the last position, past K and in the padding.  ROLLED keeps
// the branch pools' 3x3 loop rolled, for the TF32 kernel, whose four gathers in flight would otherwise need more
// registers than its two CTAs per SM leave.
template <int MODE, bool ROLLED>
__device__ __forceinline__ float4 conv_gather(const ConvPos& q, const ConvGeom& g, const ConvTap& t) {
  const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
  if (!q.img || !t.in) return zero;
  if (MODE == G_PW) return ld4(q.img + t.c);
  const int iy = q.iy0 + t.dy, ix = q.ix0 + t.dx;
  if (MODE == G_CONV3) {
    const int it = q.it0 + t.dt;
    if (it < 0 || it >= g.Tin || iy < 0 || iy >= g.Hin || ix < 0 || ix >= g.Win) return zero;
    return ld4(q.img + (((long long)it * g.Hin + iy) * g.Win + ix) * g.Cin + t.c);
  }
  if (MODE == G_CONV2) {
    if (iy < 0 || iy >= g.Hin || ix < 0 || ix >= g.Win) return zero;
    return ld4(q.img + ((long long)iy * g.Win + ix) * g.Cin + t.c);
  }
  if (MODE == G_S2MAX) {
    // the max of the 3x3 window at (2 iy, 2 ix) of the input: the (0, 0) tap, then the other eight in raster order
    if (iy < 0 || iy >= g.Hc || ix < 0 || ix >= g.Wc) return zero;
    const float* img = q.img + t.c;
    float4 v = ld4(img + ((long long)(2 * iy) * g.Win + 2 * ix) * g.Cin);
#pragma unroll
    for (int dy = 0; dy < 3; ++dy)
#pragma unroll
      for (int dx = 0; dx < 3; ++dx) {
        if (dy == 0 && dx == 0) continue;
        max4(v, ld4(img + ((long long)(2 * iy + dy) * g.Win + 2 * ix + dx) * g.Cin));
      }
    return v;
  }
  // G_BMAX / G_BAVG: the 3x3 / stride-1 / pad-1 pool around the position, in raster order
  const float init = MODE == G_BMAX ? -INFINITY : 0.f;
  float4 v = make_float4(init, init, init, init);
  int count = 0;
#pragma unroll(ROLLED ? 1 : 3)
  for (int dy = -1; dy <= 1; ++dy)
#pragma unroll(ROLLED ? 1 : 3)
    for (int dx = -1; dx <= 1; ++dx) {
      const int iy = q.iy0 + dy, ix = q.ix0 + dx;
      if (iy < 0 || iy >= g.Hin || ix < 0 || ix >= g.Win) continue;
      const float4 u = ld4(q.img + ((long long)iy * g.Win + ix) * g.Cin + t.c);
      if (MODE == G_BMAX) {
        max4(v, u);
      } else {
        v.x += u.x; v.y += u.y; v.z += u.z; v.w += u.w;
        ++count;
      }
    }
  if (MODE == G_BAVG) {
    const float d = (float)count;
    v.x /= d; v.y /= d; v.z /= d; v.w /= d;
  }
  return v;
}

}  // namespace mcvd
