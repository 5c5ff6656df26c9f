"""Run warm-up forwards, then ONE network evaluation between cudaProfilerStart/Stop (for ncu
--profile-from-start off).  usage: python tools/profile_forward.py [workload] [batch] [--kernels]

--kernels: also record that evaluation with torch.profiler and print the kernel times, the attention kernels'
share of the forward (pre-split + attention) and the CUDA-core convs' share."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from mcvd_b200 import detfill
from mcvd_b200.synthetic import make_module

kernels = "--kernels" in sys.argv
argv = [a for a in sys.argv[1:] if a != "--kernels"]
name = argv[0] if argv else "cfg2"
cfg, net, sd = make_module(name, "cuda:0")
B = int(argv[1]) if len(argv) > 1 else cfg.bench_batch
x, cond = detfill.synthetic_inputs(cfg, B)
x, cond = x.cuda(), cond.cuda()
t = torch.full((B,), 500, dtype=torch.long, device="cuda")
eng = net.engine()
P = eng.program(B)
eng.set_inputs(P, x, t, cond)
for _ in range(2):
    eng.run_cond(P)
    eng.run_step(P)
torch.cuda.synchronize()
torch.cuda.profiler.start()
eng.run_step(P)
torch.cuda.synchronize()
torch.cuda.profiler.stop()
print("ops per forward:", len(P.step_ops), "umma:", P.n_umma, "simt:", P.n_simt)
if kernels:
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        eng.run_step(P)
        torch.cuda.synchronize()
    ev = [e for e in prof.key_averages() if e.device_time_total > 0]
    total = sum(e.device_time_total for e in ev)
    share = lambda keys: sum(e.device_time_total for e in ev if any(k in e.key for k in keys)) / total
    for e in sorted(ev, key=lambda e: -e.device_time_total)[:12]:
        print(f"{e.device_time_total / 1e3:9.3f} ms {e.count:5d}x  {e.key[:110]}")
    print(f"forward kernels {total / 1e3:.3f} ms: attention {100 * share(('attention', 'attn_presplit')):.1f} %, "
          f"CUDA-core conv {100 * share(('k_conv_simt',)):.1f} %")
