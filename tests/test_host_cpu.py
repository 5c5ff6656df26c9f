"""CPU-side checks (-m "not gpu"): the oracle against the committed golden vectors (and against the
unmodified reference where MCVD_REFERENCE_ROOT names its tree), the C-ABI library's exported surface, and the host
logic that does not need a GPU."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

from common import golden, make_module, max_err, step_noise
from mcvd_b200 import arch, configs, detfill, lib, runner
from oracle import gen_golden as G, mcvd_oracle as O, ref_import

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("name", ["tiny", "tiny_spade", "tiny_rgb", "cfg1"])
def test_oracle_matches_reference_golden_forward(name):
    cfg, net, sd = make_module(name, "cpu")
    B = cfg.bench_batch
    x, cond = detfill.synthetic_inputs(cfg, B)
    g = golden(name)
    for t in (0, 37, 990):
        out = O.unet_forward(cfg, sd, x, torch.full((B,), t, dtype=torch.long), cond)
        assert max_err(out, torch.from_numpy(g[f"eps_t{t}"])) < 2e-5


@pytest.mark.parametrize("name", ["tiny", "tiny_spade"])
def test_oracle_matches_reference_golden_samplers_and_video(name):
    cfg, net, sd = make_module(name, "cpu")
    B, L = cfg.bench_batch, cfg.sampling.subsample
    x, cond = detfill.synthetic_inputs(cfg, B)
    g = golden(name)
    sched = O.make_schedule(cfg)
    fn = lambda xx, tt, cc: O.unet_forward(cfg, sd, xx, tt, cc)
    out = O.ddpm_sample(fn, sched, x.clone(), cond, L, True, True, noise=step_noise(x.shape, L))
    assert max_err(out[0], torch.from_numpy(g["ddpm"])) < 1e-3
    out = O.ddim_sample(fn, sched, x.clone(), cond, L, True, True)
    assert max_err(out[0], torch.from_numpy(g["ddim"])) < 1e-3
    out = O.fpndm_sample(fn, sched, x.clone(), cond, L, True)
    assert max_err(out[0], torch.from_numpy(g["fpndm"])) < 1e-3
    nfp = cfg.sampling.num_frames_pred
    inits = [detfill.normal(f"ar_init{i}", x.shape) for i in range(-(-nfp // cfg.data.num_frames))]
    vid = O.video_gen_loop(cfg, lambda xT, c, i: O.ddpm_sample(fn, sched, xT.clone(), c, L, True, True,
                                                               noise=step_noise(x.shape, L, tag=f"ar{i}_z")),
                           cond, inits, nfp)
    assert O.psnr01(vid, torch.from_numpy(g["video"])) > 60.0


@pytest.mark.parametrize("name", ["tiny", "tiny_spade", "cfg1"])
def test_oracle_and_module_pinned_to_live_reference(name):
    """Our module's state_dict (names, shapes, re-randomised values) and the oracle's forward against the reference
    module: as recorded in tests/golden/reference_pins.npz (oracle/gen_golden.py), and live where the tree is."""
    cfg = configs.workload(name)
    cfg2, mine, sd = make_module(name, "cpu")
    B = cfg.bench_batch
    x, cond = detfill.synthetic_inputs(cfg, B)
    t = G.pin_forward_t(B)
    ours = O.unet_forward(cfg, sd, x, t, cond)
    pins = golden("reference_pins")
    msd = mine.state_dict()
    assert list(pins[f"{name}_keys"]) == list(msd.keys())
    assert list(pins[f"{name}_sha"]) == [G.sha(sd[k]) for k in msd]          # names, dtypes, shapes and values
    assert list(pins[f"{name}_params"]) == [n for n, _ in mine.named_parameters()]   # what EMAHelper copies by
    assert max_err(ours, torch.from_numpy(pins[f"{name}_forward"])) < 2e-5
    if not ref_import.available():
        return
    ref = ref_import.build_reference_net(cfg)
    rsd = ref.state_dict()
    assert list(rsd.keys()) == list(msd.keys())
    assert all(rsd[k].shape == v.shape for k, v in msd.items())
    assert all(torch.equal(rsd[k], sd[k]) for k in rsd)
    with torch.no_grad():
        r = ref(x, t, cond=cond)
    assert max_err(ours, r) < 2e-5
    # EMA helper of the reference copies weights by parameter name into our module
    R = ref_import.ref_runner()
    ema = R.EMAHelper(mu=0.999)
    ema.register(ref)
    ema.ema(mine)
    assert all(torch.equal(p, dict(ref.named_parameters())[n]) for n, p in mine.named_parameters())


def test_library_loads_and_exports_every_declared_symbol():
    L = lib.load()
    hdr = open(os.path.join(ROOT, "include", "mcvd_b200.h")).read()
    body = hdr[hdr.index("typedef struct McvdOp"):]
    declared = set(re.findall(r"\b(mcvd_[a-z0-9_]+)\s*\(", body))
    assert declared == set(lib.EXPORTS), declared ^ set(lib.EXPORTS)
    for sym in declared:
        assert hasattr(L, sym), sym
    assert L.mcvd_abi_version() == lib.ABI_VERSION
    assert L.mcvd_sizeof_op() == ctypes.sizeof(lib.McvdOp)
    # op-kind constants of the binding == header
    for name, val in re.findall(r"(MCVD_OP_[A-Z_0-9]+)\s*=\s*(\d+)", hdr):
        py = name.replace("MCVD_", "")
        assert getattr(lib, py) == int(val), name
    for name, sh in re.findall(r"#define (MCVD_F_[A-Z_]+)\s+\(1 << (\d+)\)", hdr):
        assert getattr(lib, name.replace("MCVD_", "")) == 1 << int(sh), name


def test_validate_program_rejects_bad_ops_without_gpu():
    o = lib.McvdOp()
    o.kind, o.B = 999, 1
    with pytest.raises(RuntimeError):
        lib.validate_program(lib.make_ops([o]), 1)
    o = lib.McvdOp()
    o.kind, o.B, o.H, o.W, o.C0 = lib.OP_APPLY, 1, 4, 4, 6      # channels not a multiple of 4
    buf = torch.zeros(256)
    o.src0 = o.dst = buf.data_ptr()
    with pytest.raises(RuntimeError, match="multiples of 4"):
        lib.validate_program(lib.make_ops([o]), 1)
    # tensor-core attention needs its operand-image scratch; the size helper and the launch count are host-only
    o = lib.McvdOp()
    o.kind, o.B, o.H, o.W, o.C0, o.i0, o.i1 = lib.OP_ATTENTION_UMMA, 2, 16, 16, 192, 2, 96
    o.src0 = o.dst = buf.data_ptr()
    with pytest.raises(RuntimeError, match="scratch"):
        lib.validate_program(lib.make_ops([o]), 1)
    o.dst2 = buf.data_ptr()
    lib.validate_program(lib.make_ops([o]), 1)
    assert lib.load().mcvd_count_launches(ctypes.byref(o), 1) == 2
    assert lib.attention_scratch_bytes(2, 256, 192) == 4 * 2 * 192 * (256 + 2 * 256)
    assert lib.attention_scratch_bytes(3, 64, 32) == 4 * 3 * 32 * (128 + 2 * 64)      # Q padded to a 128-row tile


def test_product_path_fails_loudly_without_cuda():
    cfg, net, sd = make_module("tiny", "cpu")
    x, cond = detfill.synthetic_inputs(cfg, 2)
    with pytest.raises(RuntimeError, match="CUDA"):
        net(x, torch.zeros(2, dtype=torch.long), cond=cond)
    from mcvd_b200 import samplers
    with pytest.raises(RuntimeError):
        samplers.ddpm_sampler(x, net, cond=cond, subsample_steps=10)


def test_product_never_imports_oracle():
    pkg = os.path.join(ROOT, "mcvd_b200")
    for fn in os.listdir(pkg):
        if fn.endswith(".py"):
            src = open(os.path.join(pkg, fn)).read()
            assert "oracle" not in re.sub(r'""".*?"""', "", src, flags=re.S).replace("#", "\n#").split("\n#")[0] or \
                not re.search(r"^\s*(from|import)\s+oracle", src, flags=re.M), fn
            assert not re.search(r"^\s*(from|import)\s+oracle", src, flags=re.M), fn


def test_arch_spec_matches_survey_appendix_a():
    ns = arch.build_spec(configs.workload("cfg2"))
    kinds = "".join({"linear": "L", "conv3x3": "C", "res": "R", "attn": "A", "norm": "N"}[m.kind] for m in ns.mods)
    assert kinds == "LLC" + "RRR" + "RARAR" + "RARAR" + "RARA" + "RAR" + "RRRAR" + "RRRAR" + "RRRAR" + "RRR" + "NC"
    assert len(ns.mods) == 43
    assert [m.in_ch for m in ns.mods if m.kind == "res" and m.skip_ch][:4] == [768, 768, 672, 672]
    assert arch.num_groups(96) == 24 and arch.num_groups(672) == 32 and arch.num_groups(288) == 32


def test_conditioning_and_shard_helpers():
    cfg = configs.workload("tiny")
    X = torch.arange(2 * 8 * 1 * 32 * 32, dtype=torch.float32).reshape(2, 8, 1, 32, 32)
    pred, cond, mask = runner.conditioning_fn(cfg, X, num_frames_pred=5)
    assert pred.shape == (2, 5, 32, 32) and cond.shape == (2, 3, 32, 32) and mask is None
    assert torch.equal(cond, X[:, :3].reshape(2, 3, 32, 32)) and torch.equal(pred, X[:, 3:8].reshape(2, 5, 32, 32))
    if ref_import.available():
        R = ref_import.ref_runner()
        p2, c2, m2 = R.conditioning_fn(cfg, X, num_frames_pred=5)
        assert torch.equal(p2, pred) and torch.equal(c2, cond) and m2 is None
    covered = []
    for r in range(3):
        lo, hi = runner.shard_range(64, r, 3)
        covered += list(range(lo, hi))
    assert covered == list(range(64))
    assert runner.shard_range(4, 7, 8) == (4, 4)


@pytest.mark.parametrize("p_cond,p_fut,sync", list(G.MASK_CASES))
def test_conditioning_masks_match_reference_draw_for_draw(p_cond, p_fut, sync):
    """Past / future masking of the paper's "general" models (reference runner:104-147): same Bernoulli draws in
    the same order, so a seeded run of either implementation returns identical tensors -- checked against the
    reference's recorded outputs (tests/golden/reference_pins.npz), and live where the tree is."""
    cfg, X = G.mask_setup(p_cond, p_fut, sync)
    torch.manual_seed(7)
    p1, c1, m1 = runner.conditioning_fn(cfg, X, num_frames_pred=cfg.data.num_frames, prob_mask_cond=p_cond,
                                        prob_mask_future=p_fut)
    assert c1.shape[1] == cfg.data.channels * (3 + 2)
    u1 = runner.conditioning_fn(cfg, X, conditional=False)
    assert u1[1] is None and u1[2] is None
    pins, k = golden("reference_pins"), G.mask_key(p_cond, p_fut, sync)
    assert G.sha(p1) == str(pins[f"{k}_pred"]) and G.sha(c1) == str(pins[f"{k}_cond"])
    assert (m1 is None) == (f"{k}_mask" not in pins.files)
    assert m1 is None or np.array_equal(m1.numpy(), pins[f"{k}_mask"])
    # unconditional models get every frame as the prediction target
    assert G.sha(u1[0]) == str(pins[f"{k}_uncond"])
    if not ref_import.available():
        return
    R = ref_import.ref_runner()
    torch.manual_seed(7)
    p0, c0, m0 = R.conditioning_fn(cfg, X, num_frames_pred=cfg.data.num_frames, prob_mask_cond=p_cond,
                                   prob_mask_future=p_fut)
    assert torch.equal(p0, p1) and torch.equal(c0, c1)
    assert (m0 is None and m1 is None) or torch.equal(m0, m1)
    assert torch.equal(R.conditioning_fn(cfg, X, conditional=False)[0], u1[0])


def _stub_reference(tmp_path):
    """A stand-in with the reference's module layout (runners.ncsn_runner.get_model, models.{ddpm,ddim,FPNDM}_sampler,
    reference runners/ncsn_runner.py:180, models/__init__.py:39,103,207): its model is a CPU torch module, its
    samplers return a recognisable function of their inputs."""
    (tmp_path / "runners").mkdir()
    (tmp_path / "models").mkdir()
    (tmp_path / "runners" / "__init__.py").write_text("")
    (tmp_path / "models" / "__init__.py").write_text(
        "import torch\n"
        "def ddpm_sampler(x_mod, scorenet, cond=None, **kw):\n    return (x_mod * 2 + cond.sum()).unsqueeze(0)\n"
        "def ddim_sampler(x_mod, scorenet, **kw):\n    return 'reference ddim'\n"
        "def FPNDM_sampler(x_mod, scorenet, **kw):\n    return 'reference fpndm'\n")
    (tmp_path / "runners" / "ncsn_runner.py").write_text(
        "import torch\nfrom models import ddpm_sampler, ddim_sampler, FPNDM_sampler\n"
        "def get_model(config):\n    return torch.nn.Linear(2, 2)\n")


def test_patch_shim_installs_and_falls_back_on_cpu(tmp_path, monkeypatch):
    """mcvd_b200.patch swaps get_model / samplers inside the unmodified reference; on a CPU config it
    must hand back the reference module and the reference samplers' behaviour.  Runs against the real reference
    where MCVD_REFERENCE_ROOT names it, else against a stub with the reference's module layout."""
    import sys
    live = ref_import.available()
    if live:
        R = ref_import.ref_runner()
        import models as M
    else:
        _stub_reference(tmp_path)
        monkeypatch.syspath_prepend(str(tmp_path))
        for m in ("runners", "runners.ncsn_runner", "models"):
            monkeypatch.delitem(sys.modules, m, raising=False)
        import runners.ncsn_runner as R
        import models as M
    from mcvd_b200 import patch
    orig = (R.get_model, M.ddpm_sampler, M.ddim_sampler, M.FPNDM_sampler)
    try:
        patch.install(verbose=False)
        assert R.get_model is not orig[0] and M.ddpm_sampler is not orig[1] and R.ddpm_sampler is M.ddpm_sampler
        cfg = configs.workload("tiny")
        cfg.device = torch.device("cpu")
        net = R.get_model(cfg)
        assert type(net).__module__.startswith("models.better" if live else "torch.nn"), type(net)
        net.eval()
        x, cond = detfill.synthetic_inputs(cfg, 2)
        z = detfill.normal("z", x.shape)
        a = M.ddpm_sampler(x.clone(), net, cond=cond, final_only=True, subsample_steps=4, same_noise=True, noise_val=z)
        b = orig[1](x.clone(), net, cond=cond, final_only=True, subsample_steps=4, same_noise=True, noise_val=z)
        assert torch.equal(a, b)
    finally:
        R.get_model, M.ddpm_sampler, M.ddim_sampler, M.FPNDM_sampler = orig
        if not live:
            for m in ("runners", "runners.ncsn_runner", "models"):
                sys.modules.pop(m, None)


def test_metrics_oracle_grey_conversion_and_ssim_properties():
    """oracle/metrics_oracle.py (checker of MCVD_OP_FRAME_METRICS): the 8-bit grey conversion equals what
    torchvision's ToPILImage + PIL's convert('RGB').convert('L') produce (reference runners/ncsn_runner.py:1590-1599),
    and the SSIM restatement has the properties of skimage's (1 on identical images, symmetric, < 1 otherwise)."""
    import numpy as np
    from oracle import metrics_oracle as M
    rng = np.random.RandomState(0)
    for C in (1, 3):
        fr = rng.rand(C, 32, 32).astype(np.float32)
        fr[0, 0, :4] = [0.0, 1.0, 0.5, 0.999]
        try:
            from PIL import Image
            u8 = (torch.from_numpy(fr).mul(255).byte()).numpy()            # torchvision ToPILImage for float tensors
            img = Image.fromarray(u8[0], mode="L") if C == 1 else Image.fromarray(np.transpose(u8, (1, 2, 0)), mode="RGB")
            want = np.asarray(img.convert("RGB").convert("L"))
            assert np.array_equal(M.to_grey_u8(fr), want)
        except ImportError:
            pass
        g = M.to_grey_u8(fr)
        assert g.dtype == np.uint8 and g.shape == (32, 32)
    a = (rng.rand(40, 40) * 255).astype(np.uint8)
    b = np.clip(a.astype(np.int32) + rng.randint(-20, 20, a.shape), 0, 255).astype(np.uint8)
    assert abs(M.ssim_u8(a, a) - 1.0) < 1e-12
    s_ab, s_ba = M.ssim_u8(a, b), M.ssim_u8(b, a)
    assert abs(s_ab - s_ba) < 1e-12 and 0.0 < s_ab < 1.0
    pf = np.zeros((6, 4, 2))
    pf[..., 0] = rng.rand(6, 4) * 0.01 + 1e-4
    pf[..., 1] = rng.rand(6, 4)
    mse, psnr, ssim = M.best_of_repeats(pf, 3)
    assert mse.shape == (2,) and np.allclose(mse[0], pf[:3, :, 0].mean(1).min())
    assert np.allclose(psnr[1], (10 * np.log10(1 / pf[3:, :, 0].mean(1))).max()) and np.allclose(ssim[0], pf[:3, :, 1].mean(1).max())
