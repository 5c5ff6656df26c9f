"""Drop-in shim: make the UNMODIFIED reference (``main.py --config ... --video_gen`` and ``--test``,
``load_model_from_ckpt.py``, the demo notebook) use the H100 path.

    import mcvd_b200.patch; mcvd_b200.patch.install()      # before NCSNRunner / load_model are used

``get_model`` and the three samplers are plain module attributes in the reference
(``runners/ncsn_runner.py:180`` imported from ``models``; ``load_model_from_ckpt.py`` does
``from runners.ncsn_runner import get_model`` and ``from models import ddpm_sampler, ...``), so they can
be replaced without touching the reference tree.  Gamma-noise models (``model.gamma``) get the fast
model and the fast samplers, which draw the Gamma noise on the GPU.  Configurations the fast path does not
cover (3-D archs, ``noise_in_cond``, ``cond_emb``, ``output_all_frames``, SMLD, CPU devices) keep the
reference implementation: same results, no acceleration.  ``torch.nn.DataParallel`` wrappers are
accepted (the samplers unwrap ``.module``), but multi-GPU runs should use ``runner.video_gen_sharded``
(one process per GPU) instead of DataParallel's per-call weight broadcast.

The test loss ``losses.dsm.anneal_dsm_score_estimation`` (and the name ``runners.ncsn_runner`` imported) is
rebound too: a native network evaluated with grad mode off and without ``all_frames`` (``NCSNRunner.test``) gets the
native loss (``mcvd_b200.dsm``), whose noise is drawn in-kernel; every other call -- reference models, training, which
needs gradients -- keeps the reference function.

``evaluation.fid_PR.get_fid``, ``get_fid_PR`` and ``get_PR`` (and the names ``runners.ncsn_runner`` imported, used by
``--fast_fid`` and ``--sample`` with ``sampling.fid``) are rebound to ``mcvd_b200.fid``: Inception features and
k-NN precision / recall on the GPU, without the N x N host matrices.  The native version runs when the FID weights
(``pt_inception-2015-12-05-6726825d.pth``) are in the torch hub cache (``torch.hub.get_dir()/checkpoints``, where
the reference's download puts them), ``dims == 2048`` and the device is CUDA; otherwise the reference function runs.
The native path never downloads.
"""
from __future__ import annotations

import functools
import sys

from . import arch


def install(verbose: bool = True):
    import torch
    import runners.ncsn_runner as R               # the reference must be importable (on sys.path)
    import models as M
    from . import model as fast_model, samplers as fast

    ref_get_model = R.get_model
    ref_samplers = {"ddpm_sampler": M.ddpm_sampler, "ddim_sampler": M.ddim_sampler, "FPNDM_sampler": M.FPNDM_sampler}

    def get_model(config):
        dev = torch.device(getattr(config, "device", "cpu"))
        why = arch.check_supported(config) if dev.type == "cuda" else "device is not CUDA"
        if why is None:
            return fast_model.get_model(config)
        if verbose:
            print(f"[mcvd_b200] falling back to the reference model: {why}", file=sys.stderr)
        return ref_get_model(config)

    def dispatch(name):
        ref_fn, fast_fn = ref_samplers[name], getattr(fast, name)

        @functools.wraps(ref_fn)
        def sampler(x_mod, scorenet, *a, **kw):
            net = scorenet.module if hasattr(scorenet, "module") else scorenet
            is_fast = isinstance(net, fast_model.UNetMore_DDPM)
            if is_fast and not x_mod.is_cuda and next(net.parameters()).device.type != "cuda":
                raise RuntimeError("mcvd_b200 module on a CPU device: the fast path is CUDA (sm_90a) only and has "
                                   "no CPU fallback; build the reference model for CPU runs")
            use_fast = is_fast
            return (fast_fn if use_fast else ref_fn)(x_mod, scorenet, *a, **kw)
        return sampler

    R.get_model = get_model
    try:
        import losses.dsm as LD
    except ImportError:                           # a tree without the training code: nothing to rebind
        LD = None
    if LD is not None:
        from . import dsm as fast_dsm
        ref_dsm = LD.anneal_dsm_score_estimation

        @functools.wraps(ref_dsm)
        def anneal_dsm_score_estimation(scorenet, *a, **kw):
            net = scorenet.module if hasattr(scorenet, "module") else scorenet
            # all_frames is the reference signature's 10th parameter: (scorenet, x, labels, loss_type, hook, cond,
            # cond_mask, gamma, L1, all_frames)
            all_frames = kw.get("all_frames", a[8] if len(a) > 8 else False)
            if isinstance(net, fast_model.UNetMore_DDPM) and not torch.is_grad_enabled() and not all_frames:
                return fast_dsm.anneal_dsm_score_estimation(scorenet, *a, **kw)
            return ref_dsm(scorenet, *a, **kw)
        LD.anneal_dsm_score_estimation = anneal_dsm_score_estimation
        if hasattr(R, "anneal_dsm_score_estimation"):
            R.anneal_dsm_score_estimation = anneal_dsm_score_estimation
    try:
        import evaluation.fid_PR as EF
    except ImportError:                           # a tree without the evaluation code: nothing to rebind
        EF = None
    if EF is not None:
        from . import fid as fast_fid

        def fid_dispatch(name):
            ref_fn, fast_fn = getattr(EF, name), getattr(fast_fid, name)

            @functools.wraps(ref_fn)
            def fn(*a, **kw):
                # (real | path1, fake | path2, device, batch_size, dims, ...) in all three signatures
                device = kw.get("device", a[2] if len(a) > 2 else "cuda")
                dims = kw.get("dims", a[4] if len(a) > 4 else 2048)
                why = fast_fid.native_unsupported(device, dims)
                if why is None:
                    return fast_fn(*a, **kw)
                if verbose:
                    print(f"[mcvd_b200] {name}: falling back to the reference: {why}", file=sys.stderr)
                return ref_fn(*a, **kw)
            return fn
        for name in ("get_fid", "get_fid_PR", "get_PR"):
            fn = fid_dispatch(name)
            setattr(EF, name, fn)
            if hasattr(R, name):
                setattr(R, name, fn)
    for name in ref_samplers:
        fn = dispatch(name)
        setattr(M, name, fn)
        if hasattr(R, name):
            setattr(R, name, fn)
    for modname in ("load_model_from_ckpt",):
        mod = sys.modules.get(modname)
        if mod is not None:
            mod.get_model = get_model
            for name in ref_samplers:
                if hasattr(mod, name):
                    setattr(mod, name, getattr(M, name))
    return get_model
