"""Op-by-op replay of a lowered program against a float64 twin.  TEST INFRASTRUCTURE ONLY.

``Engine(module, _test_backend=Interpreter(torch.float64))`` lowers the same network with the same decisions as the
real engine (only weight packing goes through the backend), so its program pairs with the real one op for op: every
field is equal except ``w`` (fp32 taps instead of packed weight images) and, for the tensor-core convs, ``f1`` (1.0).
``replay_program`` runs the real program one op at a time; before each op it copies the real engine's current contents
of every buffer the op reads into the twin's paired buffers, so each op is judged on its exact inputs (errors do not
accumulate) and a failure names one op.

Comparisons (``err`` / ``bound`` <= 1 per element; the worst ratio per op kind is reported):
  * layout ops (NCHW_TO_NHWC, NHWC_TO_NCHW, RESIZE_NEAREST, COPY): bit-exact;
  * GN_FINALIZE: mean and rstd within 2 fp32 ulp of the float64 reference (rstd*G of the planar table within 3),
    G and S exact;
  * conv-epilogue statistics: exact int64 equality with the statistics of the conv's own stored output;
  * every other kind: |out - ref| <= TAU[kind] * A + u * |ref|, with A the op evaluated in float64 on absolute values
    (``Interpreter.exec(magnitude=True)``) and u the unit roundoff of the stored type (2^-23 covers the rounding of
    both the reference and the kernel to fp32).
"""
from __future__ import annotations

import ctypes as C

import torch

from mcvd_b200 import lib
from mcvd_b200.lib import McvdOp
from mcvd_b200.program import Engine
from op_interpreter import MAGNITUDE_KINDS, Interpreter, tile_geometry, tile_slots, tile_stats

KIND_NAME = {v: k[3:] for k, v in vars(lib).items() if k.startswith("OP_") and isinstance(v, int)}

# Per-element error bound relative to A.  The tensor-core kinds carry each operand as an fp16 hi/lo pair (about 22
# significant bits) with fp32 accumulation: on the H100 their worst error is about 0.3 of this bound at the benchmark
# workloads, while dropping one of the three partial products exceeds it about 20-fold.  APPLY (SiLU, 16-tap FIR),
# TIMESTEP_EMBED (sin/cos of an fp32 product) and DIFFUSION_UPDATE get a few fp32 ulp of the magnitude of their terms.
TAU_MATMUL = 1e-5
TAU = {lib.OP_CONV_UMMA: TAU_MATMUL, lib.OP_CONV_UMMA2: TAU_MATMUL, lib.OP_CONV_SIMT: TAU_MATMUL,
       lib.OP_CONV_SMALLN: TAU_MATMUL, lib.OP_LINEAR: TAU_MATMUL, lib.OP_ATTENTION: TAU_MATMUL,
       lib.OP_ATTENTION_UMMA: TAU_MATMUL,
       lib.OP_APPLY: 16 * 2.0 ** -24, lib.OP_TIMESTEP_EMBED: 8 * 2.0 ** -24, lib.OP_DIFFUSION_UPDATE: 8 * 2.0 ** -24,
       lib.OP_GN_PARTIAL: 1e-12}
LAYOUT_KINDS = (lib.OP_NCHW_TO_NHWC, lib.OP_NHWC_TO_NCHW, lib.OP_RESIZE_NEAREST, lib.OP_COPY)
TC_CONV_KINDS = (lib.OP_CONV_UMMA, lib.OP_CONV_UMMA2)
PTR_FIELDS = ("src0", "src1", "src2", "src3", "w", "bias", "aux0", "aux1", "aux2", "dst", "dst2")
IN_FIELDS = ("src0", "src1", "src2", "src3", "bias", "aux0", "aux1", "aux2")
VALUE_FIELDS = ("kind", "flags", "B", "H", "W", "C0", "C1", "C2", "C3", "Cout") + tuple(f"i{i}" for i in range(8)) + \
    tuple(f"f{i}" for i in range(8))


class HarnessError(AssertionError):
    """the two programs do not pair up: a fault of the replay, not of a kernel"""


def twin_engine(real: Engine, module) -> Engine:
    """the float64 interpreter twin of ``real``, with the same lowering settings"""
    twin = Engine(module, _test_backend=Interpreter(torch.float64))
    for a in ("conv_mode", "epilogue_stats", "attn_mode", "fuse_shortcut", "split_mode"):
        setattr(twin, a, getattr(real, a))
    return twin


def _tensors(eng: Engine, P) -> dict:
    out = {}

    def add(v):
        if isinstance(v, torch.Tensor):
            out.setdefault(v.data_ptr(), v)
        elif isinstance(v, (tuple, list)):
            for e in v:
                add(e)
    add(P.keep)
    add(list(eng.packed.values()))
    return out


def _outputs(op):
    """(field, elements written, dtype) of every buffer an op writes"""
    k, B, H, W = op.kind, op.B, op.H, op.W
    f32, f64 = torch.float32, torch.float64
    if k == lib.OP_NCHW_TO_NHWC:
        return [("dst", B * H * W * (op.Cout if op.Cout > 0 else op.C0 + op.C1), f32)]
    if k in (lib.OP_NHWC_TO_NCHW, lib.OP_DIFFUSION_UPDATE):
        return [("dst", B * op.C0 * H * W, f32)]
    if k in (lib.OP_TIMESTEP_EMBED, lib.OP_LINEAR):
        return [("dst", B * op.Cout, f32)]
    if k == lib.OP_GN_PARTIAL:
        return [("dst", B * op.i0 * (op.C0 + op.C1) * 2, f64)]
    if k == lib.OP_GN_FINALIZE:
        C = op.C0 + op.C1
        return [("dst", B * C * 4, f32)] + ([("dst2", B * 3 * C, f32)] if op.dst2 else [])
    if k == lib.OP_APPLY:
        n = B * H * W * (op.C0 + op.C1)
        return [("dst", n, f32)] + ([("dst2", n, f32)] if op.dst2 else [])
    if k in (lib.OP_CONV_SIMT, lib.OP_CONV_UMMA, lib.OP_CONV_UMMA2, lib.OP_CONV_SMALLN):
        out = [("dst", B * H * W * op.Cout, f32)]
        if k in TC_CONV_KINDS and op.dst2:
            pimg, nj, ntiles = tile_geometry(B, H, W, op.i0)
            out.append(("dst2", ntiles * nj * 2 * op.Cout, torch.int64))
        return out
    if k in (lib.OP_ATTENTION, lib.OP_ATTENTION_UMMA, lib.OP_RESIZE_NEAREST):
        return [("dst", B * H * W * op.C0, f32)]
    if k == lib.OP_COPY:
        return [("dst", op.i0, f32)]
    raise NotImplementedError(KIND_NAME.get(k, k))


def _ulp(x):
    """fp32 ulp of |x|"""
    a = x.float().abs()
    return (torch.nextafter(a, torch.full_like(a, float("inf"))) - a).double()


class Replay:
    def __init__(self, real: Engine, P, twin: Engine, Q):
        self.real, self.P, self.twin, self.Q = real, P, twin, Q
        self.rt, self.tt = _tensors(real, P), _tensors(twin, Q)
        self.pmap = {}
        self.stats = {}                  # kind name -> [ops replayed, worst err / bound]
        self.failures = []
        self.range_max = {}              # op label -> max |x| of a statistics-writing conv output

    # -- pairing -----------------------------------------------------------------------------------
    def _map(self, where, i, f, rp, tp):
        if not rp or not tp:
            if bool(rp) != bool(tp):
                raise HarnessError(f"{where}[{i}].{f}: one side is NULL ({rp}, {tp})")
            return
        if rp not in self.rt or tp not in self.tt:
            raise HarnessError(f"{where}[{i}].{f}: pointer is not the start of a program or packed tensor")
        if self.pmap.setdefault(rp, tp) != tp:
            raise HarnessError(f"{where}[{i}].{f}: real buffer maps to two twin buffers")

    def pair(self, where, rops, tops):
        if len(rops) != len(tops):
            raise HarnessError(f"{where}: {len(rops)} real ops, {len(tops)} twin ops")
        for i in range(len(rops)):
            self._pair_op(where, i, rops[i], tops[i])

    def _pair_op(self, where, i, r, t):
        for f in VALUE_FIELDS:
            if f == "f1" and r.kind in TC_CONV_KINDS:
                continue
            if getattr(r, f) != getattr(t, f):
                raise HarnessError(f"{where}[{i}] {KIND_NAME.get(r.kind)}: field {f} differs "
                                   f"({getattr(r, f)} vs {getattr(t, f)})")
        for f in PTR_FIELDS:
            self._map(where, i, f, getattr(r, f) or 0, getattr(t, f) or 0)

    # -- buffers -----------------------------------------------------------------------------------
    def rbuf(self, op, f, n=None):
        v = self.rt[getattr(op, f)].view(-1)
        return v if n is None else v[:n]

    def tbuf(self, op, f, n=None):
        v = self.tt[getattr(op, f)].view(-1)
        return v if n is None else v[:n]

    def _load_inputs(self, r, t):
        fields = [f for f in IN_FIELDS if getattr(r, f)] + (["dst"] if r.kind == lib.OP_DIFFUSION_UPDATE else [])
        for f in fields:
            a, b = self.rbuf(r, f), self.tbuf(t, f)
            if a.dtype != b.dtype or a.numel() != b.numel():
                raise HarnessError(f"{KIND_NAME[r.kind]}.{f}: paired buffers differ in type or size")
            if a.data_ptr() != b.data_ptr():
                b.copy_(a)

    def _run_real(self, arr, i):
        if self.real.backend is not None:
            self.real.backend.exec(arr[i])
            return
        one = (McvdOp * 1).from_address(C.addressof(arr) + i * C.sizeof(McvdOp))
        lib.run_program(one, 1, self.real._stream())
        torch.cuda.synchronize(self.real.device)

    # -- one op ------------------------------------------------------------------------------------
    def op(self, where, i, rarr, tarr):
        r, t = rarr[i], tarr[i]
        self._pair_op(where, i, r, t)
        k = r.kind
        outs = _outputs(r)
        self._load_inputs(r, t)
        for f, n, dt in outs:                       # what the kernel does not write stays visible
            if not (k == lib.OP_DIFFUSION_UPDATE and f == "dst") and not (k == lib.OP_ATTENTION_UMMA and f == "dst2"):
                self.rbuf(r, f, n).fill_(-7 if dt == torch.int64 else float("nan"))
        self._run_real(rarr, i)
        self.twin.backend.exec(t)
        ref = {f: self.tbuf(t, f, n).clone() for f, n, _ in outs}
        mag = None
        if k in MAGNITUDE_KINDS:
            self._load_inputs(r, t)
            self.twin.backend.exec(t, magnitude=True)
            mag = {f: self.tbuf(t, f, n).clone() for f, n, dt in outs if dt != torch.int64}
        label = f"{where}[{i}] {KIND_NAME[k]}"
        for f, n, dt in outs:
            got = self.rbuf(r, f, n)
            if dt == torch.int64:
                self._check_stats(label, r, got)
            elif k in LAYOUT_KINDS:
                self._record(label, r, f, 0.0 if torch.equal(got, ref[f]) else float("inf"), got, ref[f])
            elif k == lib.OP_GN_FINALIZE:
                self._check_finalize(label, r, f, got, ref[f])
            else:
                u = 2.0 ** -52 if dt == torch.float64 else 2.0 ** -23
                bound = TAU[k] * mag[f].double() + u * ref[f].double().abs()
                self._ratio(label, r, f, got, ref[f], bound)

    # -- checks ------------------------------------------------------------------------------------
    def _ratio(self, label, r, f, got, ref, bound):
        err = (got.double() - ref.double()).abs()
        ratio = torch.where(err == 0, torch.zeros_like(err), err / bound)
        ratio = torch.nan_to_num(ratio, nan=float("inf"))
        j = int(ratio.argmax())
        self._record(label, r, f, float(ratio[j]), got, ref, j, float(bound[j]))

    def _check_finalize(self, label, r, f, got, ref):
        B, C = r.B, r.C0 + r.C1
        if f == "dst":               # [B][C][4] = mean | rstd | G | S
            g, e = got.view(B, C, 4), ref.view(B, C, 4)
            k_ulp = torch.tensor([2.0, 2.0, 0.0, 0.0], dtype=torch.float64, device=got.device)
        else:                        # planar [B][3][C] = mean | rstd*G | S
            g, e = got.view(B, 3, C).transpose(1, 2), ref.view(B, 3, C).transpose(1, 2)
            k_ulp = torch.tensor([2.0, 3.0, 0.0], dtype=torch.float64, device=got.device)
        bound = (k_ulp * _ulp(e)).reshape(-1)
        self._ratio(label, r, f, g.reshape(-1), e.reshape(-1), bound)

    def _check_stats(self, label, r, got):
        y = self.rbuf(r, "dst", r.B * r.H * r.W * r.Cout).view(r.B, r.H, r.W, r.Cout)
        self.range_max[label] = float(y.abs().max())
        try:
            exp = tile_stats(y, r.i0)
        except ValueError as e:
            self.failures.append(f"{label}: {e}; {self._describe(r)}")
            return
        _, ok = tile_slots(r.B, r.H, r.W, r.i0, got.device)      # the slots GN_FINALIZE reads
        got, exp = got.view(exp.shape)[ok].reshape(-1), exp[ok].reshape(-1)
        self._record(label, r, "dst2", 0.0 if torch.equal(got, exp) else float("inf"), got, exp)

    def _record(self, label, r, f, ratio, got, ref, j=None, bound=None):
        name = KIND_NAME[r.kind] + ("" if f == "dst" else "." + f)
        s = self.stats.setdefault(name, [0, 0.0])
        s[0] += 1
        s[1] = max(s[1], ratio)
        if ratio > 1.0:
            if j is None:
                j = int((got != ref).nonzero()[0]) if (got != ref).any() else 0
            self.failures.append(f"{label}.{f}: err/bound {ratio:.3g} at element {j}: got {float(got[j]):.9g}, "
                                 f"ref {float(ref[j]):.9g}" + ("" if bound is None else f", bound {bound:.3g}") +
                                 f"; {self._describe(r)}")

    @staticmethod
    def _describe(r):
        s = (f"B={r.B} H={r.H} W={r.W} C0={r.C0} C1={r.C1} C2={r.C2} C3={r.C3} Cout={r.Cout} "
             f"i0..i5={[getattr(r, f'i{i}') for i in range(6)]} flags={r.flags:#x} f0={r.f0:.6g}")
        if r.kind in TC_CONV_KINDS:
            info = lib.umma2_plan_info(r.H, r.W, r.i0, r.C0, r.C1, r.C2, r.C3, r.i1, bool(r.dst2))
            s += f" plan={info}"
        return s

    def release(self):
        """drop the engines and buffers, keep the report"""
        self.real = self.P = self.twin = self.Q = self.rt = self.tt = self.pmap = None

    def table(self):
        return "\n".join(f"  {k:<24} {n:>5} ops   worst err/bound {w:.3g}" for k, (n, w) in sorted(self.stats.items()))


def ddpm_update(u, step=500, n_steps=1000):
    """DDPM posterior-mean coefficients of one reverse step of the linear schedule, x0 clipped, noise injected
    (models/__init__.py:287-290,324-333)"""
    betas = torch.linspace(1e-4, 0.02, n_steps, dtype=torch.float64)
    abar = torch.cumprod(1 - betas, 0)
    a, ap, beta = float(abar[step]), float(abar[step - 1]), float(betas[step])
    u.f0, u.f1 = 1.0 / a ** 0.5, (1.0 - a) ** 0.5
    u.f2, u.f3 = ap ** 0.5 * beta / (1 - a), (1 - beta) ** 0.5 * (1 - ap) / (1 - a)
    u.f4, u.f5 = 0.0, (beta * (1 - ap) / (1 - a)) ** 0.5
    u.flags = lib.F_CLIP


def replay_program(real: Engine, twin: Engine, B, x, cond, t, noise) -> Replay:
    """Replay cond ops, step ops, the NHWC -> NCHW output op and a DDPM update of the batch-B program of ``real``
    against ``twin``.  t: a float (uniform timestep) or a [B] tensor (per-clip timesteps)."""
    P, Q = real.program(B), twin.program(B)
    R = Replay(real, P, twin, Q)
    R.pair("cond", P.cond_ops, Q.cond_ops)
    R.pair("step", P.step_ops, Q.step_ops)
    R.pair("out", P.out_arr, Q.out_arr)
    R.pair("update", P.update_arr, Q.update_arr)
    for eng, prog in ((real, P), (twin, Q)):
        eng.set_inputs(prog, x=x, t=t, cond=cond)
        prog.noise.copy_(noise.reshape(prog.noise.shape))
        ddpm_update(prog.update_arr[0])
    if P.cond_arr is not None:
        for i in range(len(P.cond_ops)):
            R.op("cond", i, P.cond_arr, Q.cond_arr)
    for i in range(len(P.step_ops)):
        R.op("step", i, P.step_arr, Q.step_arr)
    eps = P.eps_nhwc.clone()
    real.run_step(P)                                      # the whole program at once: the same bits
    if real.backend is None:
        torch.cuda.synchronize(real.device)
    R.whole_program_identical = torch.equal(eps, P.eps_nhwc)
    R.op("out", 0, P.out_arr, Q.out_arr)
    R.op("update", 0, P.update_arr, Q.update_arr)
    R.n_ops = len(P.cond_ops) + len(P.step_ops) + 2
    return R
