"""CPU: the C-ABI library loads and exports every symbol include/*.h declares (no compute calls)."""
import ctypes
import glob
import os
import re

from monodetr_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    names = set()
    for h in glob.glob(os.path.join(ROOT, "include", "*.h")):
        txt = re.sub(r"/\*.*?\*/", "", open(h).read(), flags=re.S)
        names |= set(re.findall(r"\b(mdb_\w+)\s*\(", txt))
    return names


def test_library_exports_every_declared_symbol():
    assert os.path.exists(_lib.LIB_PATH), "run `python -m monodetr_b200.build` first"
    L = ctypes.CDLL(_lib.LIB_PATH)
    declared = _declared()
    assert len(declared) >= 6
    for name in sorted(declared):
        assert hasattr(L, name), f"{name} declared in include/ but not exported"


def test_loader_signatures_cover_header():
    assert _declared() == set(_lib.SIGNATURES), (_declared() ^ set(_lib.SIGNATURES))
    assert _lib.lib().mdb_abi_version() >= 1
    assert b"invalid" in _lib.lib().mdb_error_string(-1)


def test_cpu_tensor_is_rejected_loudly():
    import pytest
    import torch
    from monodetr_b200.msda import ms_deform_attn_forward
    v = torch.zeros(1, 4, 1, 4)
    sh = torch.tensor([[2, 2]]); ls = torch.tensor([0])
    loc = torch.zeros(1, 1, 1, 1, 1, 2); at = torch.zeros(1, 1, 1, 1, 1)
    with pytest.raises(RuntimeError, match="Not implemented on the CPU"):
        ms_deform_attn_forward(v, sh, ls, loc, at, 64)


def test_cpu_tensor_is_rejected_by_every_wrapper():
    """Host tensors never reach a launch: the library call names its entry point and raises before any CUDA call."""
    import pytest
    import torch
    from monodetr_b200 import functional as Fn
    n0 = _lib.launch_count()
    with pytest.raises(RuntimeError, match="mdb_box_refine_forward_f32: CUDA tensors required"):
        Fn.box_refine(torch.zeros(2, 6), torch.full((2, 2), 0.5))
    with pytest.raises(RuntimeError, match="mdb_mean3_f32: CUDA tensors required"):
        Fn.mean3(torch.zeros(8), torch.zeros(8), torch.zeros(8))
    with pytest.raises(RuntimeError, match="mdb_depth_sample_forward_f32: CUDA tensors required"):
        Fn.depth_sample(torch.zeros(1, 4, 4), torch.zeros(1, 3, 2))
    with pytest.raises(RuntimeError, match="mdb_sum_mean_squares_forward_f32: CUDA tensors required"):
        Fn.sum_mean_squares([torch.zeros(4), torch.zeros(8)])          # tensors inside a pointer array are checked too
    assert _lib.launch_count() == n0


def test_process_wide_settings_round_trip_without_a_gpu():
    """mdb_set_deterministic / mdb_set_precision are host-side switches: they answer on a machine without a GPU."""
    import monodetr_b200
    from monodetr_b200 import tc
    prev = monodetr_b200.set_deterministic(True)
    try:
        assert monodetr_b200.is_deterministic() and _lib.lib().mdb_get_deterministic() == 1
        assert monodetr_b200.set_deterministic(False) is True and not monodetr_b200.is_deterministic()
    finally:
        monodetr_b200.set_deterministic(prev)
    mode = tc.get_precision()
    assert mode in ("bf16x3", "tf32x3", "tf32")
