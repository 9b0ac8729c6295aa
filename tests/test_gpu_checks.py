"""The checks every GPU result rests on (tests/gpu_checks.py), on the CPU: each one must fail when what it guards
against happens, so that a GPU test cannot pass vacuously."""
import pytest
import torch

from fadtk_b200 import _native
from gpu_checks import Guarded, check_bound, expect_rejected

DTYPES = [torch.float16, torch.float32]


def written(dtype):
    """a [3, 5] tensor between guards of 8 and 12 elements, every element written"""
    g = Guarded((3, 5), dtype, "cpu", 8, 12)
    g.body.copy_(torch.arange(15.0).view(3, 5))
    return g


@pytest.mark.parametrize("dtype", DTYPES)
def test_fresh_buffer_is_untouched_and_unwritten(dtype):
    g = Guarded((3, 5), dtype, "cpu", 8)
    assert g.buf.numel() == 8 + 15 + 8 and g.body.shape == (3, 5)
    assert g.untouched() and g.guards_intact() and not g.fully_written()
    with pytest.raises(AssertionError, match="unwritten"):
        g.check()


@pytest.mark.parametrize("dtype", DTYPES)
def test_written_body_passes(dtype):
    g = written(dtype)
    assert g.check() is g.body
    assert not g.untouched()


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("where", [0, 7, 8 + 15, 8 + 15 + 11])
def test_write_into_a_guard_fails(dtype, where):
    g = written(dtype)
    g.buf[where] = 1.0
    assert not g.guards_intact()
    with pytest.raises(AssertionError, match="guard"):
        g.check()


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("where", [(0, 0), (2, 4)])
def test_element_left_unwritten_fails(dtype, where):
    g = written(dtype)
    g.body.view(g.idt)[where] = g.bits
    assert g.guards_intact() and not g.fully_written()
    with pytest.raises(AssertionError, match="unwritten"):
        g.check()


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("value", [float("nan"), float("inf"), -float("inf")])
def test_non_finite_value_fails(dtype, value):
    g = written(dtype)
    g.body[1, 2] = value
    assert g.guards_intact() and g.fully_written()
    with pytest.raises(AssertionError, match="non-finite"):
        g.check()


@pytest.mark.parametrize("dtype", DTYPES)
def test_modified_input_is_not_intact(dtype):
    g = Guarded((3, 5), dtype, "cpu", 8, init=torch.ones((3, 5)))
    assert g.intact_input() and g.fully_written()
    g.body[0, 0] = 2.0
    assert not g.intact_input()
    g.body[0, 0] = 1.0
    g.buf[-1] = 0.0
    assert not g.intact_input()


@pytest.mark.parametrize("dtype", DTYPES)
def test_pointer_kinds(dtype):
    g = Guarded((3, 5), dtype, "cpu", 8)
    assert g.ptr("ok") is g.body and g.ptr("null") is None
    assert g.ptr("odd").data_ptr() == g.body.data_ptr() + g.body.element_size()


# ------------------------------------------------------------------------------------------------ rejected calls
class StubEngine:
    launches = 0


def rejected(message, write=False, launch=False):
    def call(engine, outs):
        o = Guarded((4,), torch.float32, "cpu", 8)
        outs.append(o)
        if write:
            o.body[3] = 0.0
        if launch:
            engine.launches += 1
        raise _native.NativeError(message)
    return call


def test_rejected_call_passes():
    expect_rejected(StubEngine(), rejected("entry: bad"), "entry: bad", [])


def test_rejected_call_that_writes_fails():
    with pytest.raises(AssertionError, match="wrote output"):
        expect_rejected(StubEngine(), rejected("entry: bad", write=True), "entry: bad", [])


def test_rejected_call_that_launches_fails():
    with pytest.raises(AssertionError, match="launched a kernel"):
        expect_rejected(StubEngine(), rejected("entry: bad", launch=True), "entry: bad", [])


def test_other_message_fails():
    with pytest.raises(AssertionError, match="want 'entry: bad'"):
        expect_rejected(StubEngine(), rejected("entry: worse"), "entry: bad", [])


def test_accepted_call_fails():
    with pytest.raises(pytest.fail.Exception):
        expect_rejected(StubEngine(), lambda engine, outs: None, "entry: bad", [])


# ------------------------------------------------------------------------------------------------- error bounds
def test_check_bound():
    ref = torch.tensor([1.0, -2.0, 4.0], dtype=torch.float64)
    got = (ref + torch.tensor([1e-3, 0.0, -1e-3], dtype=torch.float64)).float()
    stats = {}
    rms, ratio = check_bound("k", "first", got, ref, torch.full_like(ref, 2e-3), stats, {"k": 1e-3})
    assert 0.4 < ratio < 0.6 and 0 < rms < 1e-3
    assert stats == {"k": [rms, ratio, "first"]}
    with pytest.raises(AssertionError, match="bound"):
        check_bound("k", "over the bound", got, ref, torch.full_like(ref, 5e-4), stats, {})
    with pytest.raises(AssertionError, match="rms relative error"):
        check_bound("k", "over the ceiling", got, ref, torch.full_like(ref, 2e-3), stats, {"k": 1e-4})
    check_bound("other", "no ceiling", got, ref, torch.full_like(ref, 2e-3), stats, {"k": 1e-4})
    assert stats["other"][2] == "no ceiling"
