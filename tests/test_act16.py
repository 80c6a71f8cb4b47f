"""The 16-bit activation arguments of the C ABI, CPU side: the plane offset the host wrappers derive from a tensor
(lib.plane16), their refusals before any launch, and the C entries' checks of (pointer, plane) pairs that reach them
without a tensor."""
import ctypes

import pytest
import torch

from fgt_b200 import lib


@pytest.fixture
def no_launch(monkeypatch):
    def refuse(name, *args, **kwargs):
        raise AssertionError(f"{name} was called")
    monkeypatch.setattr(lib, "call", refuse)


def test_plane16():
    s = lib.empty_split((6, 8), "cpu")
    assert lib.plane16(s) == 48
    assert lib.plane16(s[:, 2:4]) == 48                     # row-sliced view: same planes
    assert lib.plane16(torch.empty(6, 8, dtype=torch.float16)) == 0
    assert lib.plane16(None) == 0
    assert lib.act16_dtype(True) == torch.float16 and lib.act16_dtype(False) == torch.bfloat16
    with pytest.raises(TypeError):
        lib.plane16(torch.empty(6, 8, dtype=torch.float16), split_only=True)
    with pytest.raises(ValueError):
        lib.plane16(torch.empty(6, 8, dtype=torch.bfloat16))
    with pytest.raises(TypeError):
        lib.plane16(torch.empty(2, 8))


def test_split_only_wrappers_refuse_fp16_before_any_launch(no_launch):
    img = torch.zeros(1, 10, 10, 64)
    with pytest.raises(TypeError):
        lib.unfold(img, 1, 4, 4, 64, 7, 7, 3, 3, 10, 10, torch.empty(16, 49 * 64, dtype=torch.float16))
    with pytest.raises(TypeError):
        lib.pack_nchw(torch.zeros(1, 3, 8, 8), None, torch.empty(1, 8, 8, 8, dtype=torch.float16))
    with pytest.raises(TypeError):
        lib.f16_to_split(torch.zeros(64, dtype=torch.float16), torch.empty(64, dtype=torch.float16))


def test_wrappers_refuse_bf16_without_its_plane_dimension(no_launch):
    img = torch.zeros(1, 10, 10, 64)
    with pytest.raises(ValueError):
        lib.unfold(img, 1, 4, 4, 64, 7, 7, 3, 3, 10, 10, torch.empty(16, 49 * 64, dtype=torch.bfloat16))
    with pytest.raises(ValueError):
        lib.pack_nchw(torch.zeros(1, 3, 8, 8), None, torch.empty(1, 8, 8, 8, dtype=torch.bfloat16))
    with pytest.raises(ValueError):
        lib.fold_unfold(torch.zeros(16, 49 * 64), 1, 4, 4, 64, 7, 7, 3, 3, 10, 10,
                        torch.empty(16, 49 * 64, dtype=torch.bfloat16))


def test_c_entries_check_planes_they_did_not_check_without_touching_the_gpu():
    L = lib.load()
    one = ctypes.c_void_p(64)   # non-null dummies; never dereferenced when validation fails first
    calls = [
        lambda: L.fgt_unfold(one, 1, 4, 4, 64, 7, 7, 3, 3, 10, 10, 1, one, 0, None),     # split-only: plane 0
        lambda: L.fgt_pack_nchw(one, 3, None, 0, 1, 8, 8, 0, 8, one, 0, None),            # split-only: plane 0
        lambda: L.fgt_raft_flow_update(one, None, 0, 1, 8, 8, one, one, -2, 128, 126, None),
    ]
    for fn in calls:
        assert fn() == -1                           # FGT_ERR_ARG
        assert "plane offset" in L.fgt_last_error().decode(), L.fgt_last_error()
