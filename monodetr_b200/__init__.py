"""monodetr_b200 -- H100 (sm_90a) implementation of MonoDETR's forward/backward hot path behind the reference's
own interfaces: `build_monodetr(cfg)` / `MonoDETR.forward`, the `MSDeformAttn` module and the
`MultiScaleDeformableAttention` extension functions.  Kernels live in csrc/ behind the C ABI of
include/monodetr_b200.h (libmonodetr_b200.so, built by `python -m monodetr_b200.build`)."""


def build_monodetr(cfg, criterion_builder=None):
    """Mirror of lib/models/monodetr/__init__.py:4-5."""
    from .monodetr import build
    return build(cfg, criterion_builder)


def set_deterministic(on=True):
    """Reproducible mode (`mdb_set_deterministic`, include/monodetr_b200.h): every float accumulation of the training iteration
    runs in a fixed order (the default path, like the reference's kernel, combines partial sums with atomics), and the depth
    predictor resizes with the library's kernel instead of F.interpolate.  On the same GPU model and build, in one process, with
    the device criterion, two training iterations from the same weights, optimizer state, inputs, targets and dropout seed
    (torch.manual_seed, or kernels.reseed) give identical bits, eagerly or as a replayed CUDA graph; multi-GPU all-reduce order
    is not covered.  A test / debugging mode: 4.4x slower per training step on an H100 (DESIGN.md section 5).  Set it before the
    model is built.  Returns the previous setting."""
    from . import _lib
    prev = bool(_lib.lib().mdb_get_deterministic())
    _lib.check(_lib.lib().mdb_set_deterministic(1 if on else 0), "set_deterministic")
    return prev


def is_deterministic():
    from . import _lib
    return bool(_lib.lib().mdb_get_deterministic())


__all__ = ["build_monodetr", "set_deterministic", "is_deterministic"]
