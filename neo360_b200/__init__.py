"""neo360_b200 -- H100-native (sm_90a) implementation of NeO-360's ray-marching hot path behind the reference's
`model(rays, randomized, white_bkgd, near, far, out_depth)` call surface.  See DESIGN.md / INTEGRATION.md."""
from . import synth  # noqa: F401

__all__ = ["NeRF_TP", "NeRFPPMLP", "PixelNeRF", "ops", "mesh", "synth", "release_cached"]


def release_cached() -> None:
    """Return the device blocks the library keeps from destroyed scenes (for fast scene changes) to the driver (`neo_release_cached`)."""
    from . import _lib
    _lib.load().neo_release_cached()


def __getattr__(name):
    if name in ("NeRF_TP", "NeRFPPMLP"):
        from . import renderer
        return getattr(renderer, name)
    if name == "PixelNeRF":
        from . import pixelnerf
        return pixelnerf.PixelNeRF
    if name in ("ops", "mesh"):
        import importlib
        return importlib.import_module("." + name, __name__)
    raise AttributeError(name)
