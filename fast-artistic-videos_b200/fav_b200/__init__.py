"""fav_b200 -- host-side mirror of the reference's operator surface for the per-frame video-style-transfer
hot path, over the C ABI of libfav_b200.so (include/fav.h).  sm_90a only; no CPU fallback.

  stn.BilinearSamplerBDHW          <- stnbdhw/BilinearSamplerBDHW.lua
  utils.warp_image / min_filter    <- fast_artistic_video/utils.lua
  preprocess.vgg                   <- fast_artistic_video/preprocess.lua
  flowFileLoader.load              <- flowFileLoader.lua
  models_video.build_model         <- fast_artistic_video/models_video.lua
  core.run_fast_neural_video       <- fast_artistic_video_core.lua
  consistencyChecker.check / main  <- consistencyChecker/consistencyChecker.cpp
"""
from . import synth  # noqa: F401  (pure numpy; importable without the shared library)


def __getattr__(name):
    import importlib

    if name in ("_lib", "stn", "utils", "preprocess", "flowFileLoader", "models_video", "core", "consistencyChecker",
                "session", "video"):
        return importlib.import_module(f"{__name__}.{name}")
    raise AttributeError(name)
