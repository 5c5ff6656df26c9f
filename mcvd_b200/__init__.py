"""mcvd_b200 -- H100-native (sm_90a) implementation of the MCVD DDPM-sampling hot path.

Public surface mirrors the reference (voletiv/mcvd-pytorch): ``get_model(config)``,
``ddpm_sampler / ddim_sampler / FPNDM_sampler``, ``get_sampler(config)``, ``conditioning_fn`` and the
autoregressive ``video_gen_clips`` loop; see INTEGRATION.md for the drop-in shim.
Importing the package does not load CUDA; the C-ABI library is loaded (and built when nvcc is
present) on first use and every failure is loud -- there is no CPU fallback.
"""
from .configs import workload, namespace_from_dict  # noqa: F401

__all__ = ["workload", "namespace_from_dict", "get_model", "UNetMore_DDPM", "ddpm_sampler", "ddim_sampler",
           "FPNDM_sampler", "get_sampler", "conditioning_fn", "video_gen_clips", "video_gen_sharded"]


def __getattr__(name):  # lazy: keep `import mcvd_b200` cheap and torch-free until needed
    if name in ("get_model", "UNetMore_DDPM"):
        from . import model
        return getattr(model, name)
    if name in ("ddpm_sampler", "ddim_sampler", "FPNDM_sampler", "get_sampler"):
        from . import samplers
        return getattr(samplers, name)
    if name in ("conditioning_fn", "video_gen_clips", "video_gen_sharded", "gather_clips", "shard_range",
                "data_transform", "inverse_data_transform"):
        from . import runner
        return getattr(runner, name)
    raise AttributeError(name)
