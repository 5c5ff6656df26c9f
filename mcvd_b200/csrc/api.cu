// C-ABI entry points (include/mcvd_b200.h): program runner, validation, error reporting.
#include <stdarg.h>
#include <string.h>

#include "conv_eval.cuh"

namespace mcvd {

static thread_local char g_err[512] = {0};

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

static int dispatch(const McvdOp& op, cudaStream_t s) {
  switch (op.kind) {
    case MCVD_OP_NCHW_TO_NHWC: return launch_nchw_to_nhwc(op, s);
    case MCVD_OP_NHWC_TO_NCHW: return launch_nhwc_to_nchw(op, s);
    case MCVD_OP_TIMESTEP_EMBED: return launch_timestep_embed(op, s);
    case MCVD_OP_LINEAR: return launch_linear(op, s);
    case MCVD_OP_GN_PARTIAL: return launch_gn_partial(op, s);
    case MCVD_OP_GN_FINALIZE: return launch_gn_finalize(op, s);
    case MCVD_OP_APPLY: return launch_apply(op, s);
    case MCVD_OP_CONV_SIMT: return launch_conv_simt(op, s);
    case MCVD_OP_ATTENTION: return launch_attention(op, s);
    case MCVD_OP_RESIZE_NEAREST: return launch_resize_nearest(op, s);
    case MCVD_OP_DIFFUSION_UPDATE: return launch_diffusion_update(op, s);
    case MCVD_OP_CONV_UMMA: return launch_conv_umma(op, s);
    case MCVD_OP_CONV_UMMA2: return launch_conv_umma2(op, s);
    case MCVD_OP_CONV_SMALLN: return launch_conv_smalln(op, s);
    case MCVD_OP_COPY: return launch_copy(op, s);
    case MCVD_OP_ATTENTION_UMMA: return launch_attention_umma(op, s);
    case MCVD_OP_FRAME_METRICS: return launch_frame_metrics(op, s);
    case MCVD_OP_NOISE: return launch_noise(op, s);
    case MCVD_OP_LPIPS_PREP: return launch_lpips_prep(op, s);
    case MCVD_OP_CONV_RELU:
    case MCVD_OP_CONV3D:
    case MCVD_OP_CONV2D: return launch_conv_ffma(op, s);
    case MCVD_OP_MAXPOOL3D:
    case MCVD_OP_MAXPOOL2D: return launch_maxpool(op, s);
    case MCVD_OP_CONV3D_TF32:
    case MCVD_OP_CONV2D_TF32:
    case MCVD_OP_CONV_RELU_TF32: return launch_conv_tf32(op, s);
    case MCVD_OP_LPIPS_LAYER: return launch_lpips_layer(op, s);
    case MCVD_OP_I3D_PREP: return launch_i3d_prep(op, s);
    case MCVD_OP_I3D_HEAD: return launch_i3d_head(op, s);
    case MCVD_OP_DSM_PERTURB: return launch_dsm_perturb(op, s);
    case MCVD_OP_DSM_LOSS: return launch_dsm_loss(op, s);
    case MCVD_OP_FID_PREP: return launch_fid_prep(op, s);
    case MCVD_OP_FID_HEAD: return launch_fid_head(op, s);
    case MCVD_OP_KNN_RADIUS:
    case MCVD_OP_KNN_COVER: return launch_knn(op, s);
    default: break;
  }
  set_error("unknown op kind %d", op.kind);
  return -1;
}

static int validate_one(const McvdOp& op, int idx) {
  if (op.kind <= 0 || op.kind >= MCVD_OP__COUNT || op.kind == MCVD_OP__UNASSIGNED_36) {
    set_error("op %d: unknown kind %d", idx, op.kind);
    return -1;
  }
  if (op.B <= 0) {
    set_error("op %d (kind %d): batch %d", idx, op.kind, op.B);
    return -1;
  }
  const bool spatial = op.kind != MCVD_OP_TIMESTEP_EMBED && op.kind != MCVD_OP_LINEAR && op.kind != MCVD_OP_COPY;
  if (spatial && (op.H <= 0 || op.W <= 0)) {
    set_error("op %d (kind %d): spatial size %dx%d", idx, op.kind, op.H, op.W);
    return -1;
  }
  if (!op.dst || (!op.src0 && op.kind != MCVD_OP_NOISE)) {
    set_error("op %d (kind %d): null src0/dst", idx, op.kind);
    return -1;
  }
  if (op.C1 > 0 && !op.src1 && op.kind != MCVD_OP_DIFFUSION_UPDATE) {
    set_error("op %d (kind %d): C1=%d but src1 is null", idx, op.kind, op.C1);
    return -1;
  }
  auto misaligned = [](const void* p) { return p && (reinterpret_cast<uintptr_t>(p) & 15) != 0; };
  if (misaligned(op.src0) || misaligned(op.src1) || misaligned(op.dst) || misaligned(op.w) || misaligned(op.aux0) ||
      misaligned(op.aux1) || misaligned(op.aux2)) {
    set_error("op %d (kind %d): pointers must be 16-byte aligned", idx, op.kind);
    return -1;
  }
  switch (op.kind) {
    case MCVD_OP_APPLY:
      if (op.C0 % 4 || op.C1 % 4) {
        set_error("op %d APPLY: channels (%d,%d) not multiples of 4", idx, op.C0, op.C1);
        return -1;
      }
      break;
    case MCVD_OP_CONV_SIMT:
    case MCVD_OP_CONV_UMMA:
    case MCVD_OP_CONV_UMMA2:
      if (!op.w || (op.i0 != 1 && op.i0 != 3)) {
        set_error("op %d CONV: null weights or kernel size %d", idx, op.i0);
        return -1;
      }
      if (op.kind != MCVD_OP_CONV_SIMT && (op.flags & MCVD_F_HALF) && op.i3 != 0 && op.i3 != 3) {
        set_error("op %d CONV: MCVD_F_HALF runs one product; operand split %d must be 0 or 3", idx, op.i3);
        return -1;
      }
      break;
    case MCVD_OP_ATTENTION:
    case MCVD_OP_ATTENTION_UMMA:
      if (op.i0 * op.i1 != op.C0) {
        set_error("op %d ATTENTION: heads %d x dim %d != %d", idx, op.i0, op.i1, op.C0);
        return -1;
      }
      if (op.kind == MCVD_OP_ATTENTION_UMMA && (!op.dst2 || (reinterpret_cast<uintptr_t>(op.dst2) & 15))) {
        set_error("op %d ATTENTION_UMMA: dst2 (operand-image scratch) is null or not 16-byte aligned", idx);
        return -1;
      }
      break;
    case MCVD_OP_DIFFUSION_UPDATE:
    case MCVD_OP_NOISE:
      if (op.flags & MCVD_F_GAMMA) {
        if (op.kind == MCVD_OP_DIFFUSION_UPDATE && !(op.flags & MCVD_F_PHILOX)) {
          set_error("op %d DIFFUSION_UPDATE: MCVD_F_GAMMA needs MCVD_F_PHILOX", idx);
          return -1;
        }
        if (const char* why = gamma_params_error(op)) {
          set_error("op %d (kind %d): %s", idx, op.kind, why);
          return -1;
        }
      }
      break;
    case MCVD_OP_LPIPS_PREP:
      if (!op.src1 || !op.w) {
        set_error("op %d LPIPS_PREP: null real frames or resize table", idx);
        return -1;
      }
      if (op.C0 != 1 && op.C0 != 3) {
        set_error("op %d LPIPS_PREP: %d channels per frame (1 or 3)", idx, op.C0);
        return -1;
      }
      if (op.H != 128 || op.W != 128) {
        set_error("op %d LPIPS_PREP: output side %dx%d (must be 128x128)", idx, op.H, op.W);
        return -1;
      }
      if (op.i0 < 1 || op.i1 < 1 || op.i2 < 1 || 2LL * op.B * op.i0 > 65535) {
        set_error("op %d LPIPS_PREP: %d frames of side %d, %d taps, batch %d", idx, op.i0, op.i1, op.i2, op.B);
        return -1;
      }
      break;
    case MCVD_OP_CONV_RELU:
    case MCVD_OP_CONV3D:
    case MCVD_OP_MAXPOOL3D:
    case MCVD_OP_CONV2D:
    case MCVD_OP_MAXPOOL2D:
    case MCVD_OP_CONV3D_TF32:
    case MCVD_OP_CONV2D_TF32:
    case MCVD_OP_CONV_RELU_TF32: {
      ConvGeom g;
      const bool tf32 = op.kind == MCVD_OP_CONV3D_TF32 || op.kind == MCVD_OP_CONV2D_TF32 ||
                        op.kind == MCVD_OP_CONV_RELU_TF32;
      if (const char* why = tf32 ? conv_tf32_geom(op, g) : conv_geom(op, g)) {
        set_error("op %d %s: %s", idx, conv_kind_name(op.kind), why);
        return -1;
      }
      if (misaligned(op.bias)) {
        set_error("op %d %s: bias must be 16-byte aligned", idx, conv_kind_name(op.kind));
        return -1;
      }
      break;
    }
    case MCVD_OP_LPIPS_LAYER:
      if (!op.src1 || !op.w || op.C0 < 1) {
        set_error("op %d LPIPS_LAYER: null real features or lin weights, or %d channels", idx, op.C0);
        return -1;
      }
      break;
    case MCVD_OP_I3D_PREP:
    case MCVD_OP_I3D_HEAD: {
      const char* name = op.kind == MCVD_OP_I3D_PREP ? "I3D_PREP" : "I3D_HEAD";
      if (const char* why = op.kind == MCVD_OP_I3D_PREP ? i3d_prep_error(op) : i3d_head_error(op)) {
        set_error("op %d %s: %s", idx, name, why);
        return -1;
      }
      if (misaligned(op.bias)) {
        set_error("op %d %s: bias must be 16-byte aligned", idx, name);
        return -1;
      }
      break;
    }
    case MCVD_OP_DSM_PERTURB:
    case MCVD_OP_DSM_LOSS:
      if (const char* why = dsm_error(op)) {
        set_error("op %d %s: %s", idx, op.kind == MCVD_OP_DSM_PERTURB ? "DSM_PERTURB" : "DSM_LOSS", why);
        return -1;
      }
      break;
    case MCVD_OP_FID_PREP:
    case MCVD_OP_FID_HEAD:
    case MCVD_OP_KNN_RADIUS:
    case MCVD_OP_KNN_COVER: {
      const char* why = op.kind == MCVD_OP_FID_PREP   ? fid_prep_error(op)
                        : op.kind == MCVD_OP_FID_HEAD ? fid_head_error(op)
                                                      : knn_error(op);
      const char* name = op.kind == MCVD_OP_FID_PREP     ? "FID_PREP"
                         : op.kind == MCVD_OP_FID_HEAD   ? "FID_HEAD"
                         : op.kind == MCVD_OP_KNN_RADIUS ? "KNN_RADIUS"
                                                         : "KNN_COVER";
      if (why) {
        set_error("op %d %s: %s", idx, name, why);
        return -1;
      }
      if (misaligned(op.bias)) {
        set_error("op %d %s: bias must be 16-byte aligned", idx, name);
        return -1;
      }
      break;
    }
    default: break;
  }
  return 0;
}

}  // namespace mcvd

extern "C" {

int mcvd_abi_version(void) { return MCVD_ABI_VERSION; }
int mcvd_sizeof_op(void) { return (int)sizeof(McvdOp); }
const char* mcvd_last_error(void) { return mcvd::g_err; }

int mcvd_device_arch(void) {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) {
    cudaGetLastError();
    mcvd::set_error("no CUDA device");
    return -1;
  }
  cudaDeviceProp p;
  if (cudaGetDeviceProperties(&p, dev) != cudaSuccess) {
    cudaGetLastError();
    mcvd::set_error("cudaGetDeviceProperties failed");
    return -1;
  }
  return p.major * 10 + p.minor;
}

int mcvd_validate_program(const McvdOp* ops, int n) {
  if (!ops || n < 0) {
    mcvd::set_error("null program");
    return -1;
  }
  for (int i = 0; i < n; ++i) {
    int r = mcvd::validate_one(ops[i], i);
    if (r) return r;
  }
  return 0;
}

int mcvd_count_launches(const McvdOp* ops, int n) {
  if (!ops || n < 0) return -1;
  int total = 0;
  for (int i = 0; i < n; ++i) total += (ops[i].kind == MCVD_OP_ATTENTION_UMMA) ? 2 : 1;   // pre-split + attention
  return total;
}

int mcvd_attention_key_tile(int kind, int T, int d) {
  if (kind == MCVD_OP_ATTENTION) return mcvd::attention_simt_key_tile(T, d);
  if (kind == MCVD_OP_ATTENTION_UMMA) return mcvd::attention_umma_key_tile(T, d);
  return 0;
}

int mcvd_run_program(const McvdOp* ops, int n, void* stream) {
  if (!ops || n < 0) {
    mcvd::set_error("null program");
    return -1;
  }
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  for (int i = 0; i < n; ++i) {
    int r = mcvd::dispatch(ops[i], s);
    if (r) {
      char tmp[400];
      strncpy(tmp, mcvd::g_err, sizeof(tmp) - 1);
      tmp[sizeof(tmp) - 1] = 0;
      mcvd::set_error("op %d (kind %d): %s", i, ops[i].kind, tmp);
      return r;
    }
  }
  return 0;
}

}  // extern "C"
