"""unpack_info / unpack_data / pack_data: signatures, where the names resolve, and the argument errors that need no
GPU (shape and dtype asserts come before the CUDA check, so CPU tensors reach them)."""
import inspect

import pytest
import torch


def test_signatures_and_defaults():
    from nerfacc_b200 import pack
    assert list(inspect.signature(pack.unpack_info).parameters) == ["packed_info", "n_samples"]
    p = inspect.signature(pack.unpack_data).parameters
    assert list(p) == ["packed_info", "data", "n_samples", "pad_value"]
    assert p["n_samples"].default is None and p["pad_value"].default == 0
    assert list(inspect.signature(pack.pack_data).parameters) == ["data", "mask"]


def test_names_resolve_from_every_import_path():
    import nerfacc
    import nerfacc.pack
    import nerfacc_b200
    from nerfacc_b200 import pack
    for name in ("unpack_info", "unpack_data", "pack_data"):
        fn = getattr(pack, name)
        assert getattr(nerfacc, name) is fn and getattr(nerfacc.pack, name) is fn
        assert getattr(nerfacc_b200, name) is fn and name in nerfacc_b200.__all__


def test_cpu_tensors_raise_not_implemented():
    import nerfacc_b200 as nfa
    pi = torch.tensor([[0, 2], [2, 1]])
    with pytest.raises(NotImplementedError):
        nfa.unpack_info(pi, 3)
    with pytest.raises(NotImplementedError):
        nfa.unpack_data(pi, torch.zeros(3, 2))
    with pytest.raises(NotImplementedError):
        nfa.pack_data(torch.zeros(2, 4, 3), torch.ones(2, 4, dtype=torch.bool))


@pytest.mark.parametrize("mask", [torch.ones(2, 4, dtype=torch.uint8), torch.ones(2, 4),  # not bool
                                  torch.ones(8, dtype=torch.bool), torch.ones(2, 4, 1, dtype=torch.bool),  # not 2D
                                  torch.ones(2, 5, dtype=torch.bool)])  # does not match data
def test_pack_data_rejects_bad_masks(mask):
    import nerfacc_b200 as nfa
    with pytest.raises(AssertionError):
        nfa.pack_data(torch.zeros(2, 4, 3), mask)


@pytest.mark.parametrize("pi", [torch.zeros(4, dtype=torch.int64), torch.zeros(4, 3, dtype=torch.int64),
                                torch.zeros(2, 2, 1, dtype=torch.int64)])
def test_packed_info_must_be_n_by_2(pi):
    import nerfacc_b200 as nfa
    with pytest.raises(AssertionError):
        nfa.unpack_info(pi, 4)
    with pytest.raises(AssertionError):
        nfa.unpack_data(pi, torch.zeros(4, 2))


def test_workspace_size_is_host_code():
    from nerfacc_b200 import _lib
    assert _lib.load().nfa_chunk_order_workspace_bytes() >= 4


def test_argument_errors_do_not_need_a_gpu():
    from nerfacc_b200 import _lib
    lib = _lib.load()
    assert lib.nfa_unpack_info(-1, None, 4, None, None, None) == -1
    assert lib.nfa_unpack_info(3, None, 4, None, None, None) == -1
    assert lib.nfa_unpack_info(0, None, 4, None, None, None) == 0  # nothing to write
    assert lib.nfa_unpack_rows(2, None, 4, 3, 8, None, None, None, None) == -1
    assert lib.nfa_unpack_rows(2, None, 4, 3, -8, None, None, None, None) == -1
    assert lib.nfa_pack_rows(2, None, 4, 3, 8, None, None, None, None) == -1
    assert lib.nfa_mask_counts(2, 3, None, None, None) == -1
    assert lib.nfa_pack_masked(2, 3, 4, None, None, None, None, None) == -1
    assert lib.nfa_unpack_masked(-2, 3, 4, None, None, None, None, None) == -1
