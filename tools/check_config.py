"""Full-size functional check of a workload (mcvd_b200/configs.py) on the GPU: forward parity vs the oracle for a few clips
(+ forward time).  usage: check_config.py cfg3 [batch]"""
import os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from mcvd_b200 import detfill
from mcvd_b200.synthetic import make_module, allclose_report
from oracle import mcvd_oracle as O
name = sys.argv[1]; B = int(sys.argv[2]) if len(sys.argv) > 2 else 2
t0 = time.time()
cfg, net, sd = make_module(name, "cuda:0")
x, cond = detfill.synthetic_inputs(cfg, B)
tt = torch.tensor([500, 37][:B] + [990] * max(0, B - 2))
out = net(x.cuda(), tt.cuda(), cond=cond.cuda())
torch.cuda.synchronize()
P = net.engine().program(B)
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
for _ in range(3): net.engine().run_step(P)
e1.record(); torch.cuda.synchronize()
torch.set_num_threads(16)
ref = O.unet_forward(cfg, sd, x[:1], tt[:1], cond[:1])
bad, mx, ratio = allclose_report(out[:1].cpu(), ref, 1e-3, 1e-4)
print(f"{name}: B={B} ops/forward {len(P.step_ops)} (+{len(P.cond_ops)} cond-only) umma {P.n_umma} simt {P.n_simt}; "
      f"forward {e0.elapsed_time(e1)/3:.2f} ms; vs oracle: {bad} elements out of tol, max abs err {mx:.2e} "
      f"(ref std {ref.std():.3f}); total {time.time()-t0:.0f}s", flush=True)
assert bad == 0
