"""CPU: how deform_network.forward reads times_sel (deformation.classify_times) -- one time for every row (a number, a
one-element tensor, or equal elements without grad: the collapsed-time-row path), one time per row (any other tensor of N
elements: the per-row path), or refused (any other element count) -- before anything reaches the GPU."""
import importlib

import pytest
import torch

d = importlib.import_module("4dgaussians_b200.deformation")


def test_numbers_and_one_element_tensors_are_one_time():
    assert d.classify_times(0, 5) == (0.0, None)
    assert d.classify_times(0.25, 5) == (0.25, None)
    assert d.classify_times(torch.tensor(0.5), 5) == (0.5, None)
    assert d.classify_times(torch.tensor([[0.75]], requires_grad=True), 5) == (0.75, None)
    with pytest.raises(RuntimeError):
        d.classify_times(None, 5)


def test_equal_rows_without_grad_are_one_time_in_any_dtype_and_count():
    assert d.classify_times(torch.tensor(0.75).repeat(7, 1), 7) == (0.75, None)
    assert d.classify_times(torch.zeros(3, 1, dtype=torch.int64), 3) == (0.0, None)
    assert d.classify_times(torch.full((4,), -0.5, dtype=torch.float64), 9) == (-0.5, None)   # as before: row 0's time
    assert d.classify_times(torch.zeros(0), 0) == (0.0, None)


def test_rows_that_differ_or_require_grad_are_per_row():
    for t in (torch.linspace(-1, 1, 6), torch.linspace(-1, 1, 6).reshape(6, 1).double(), torch.arange(6) % 2,
              torch.full((6, 1), 0.3, requires_grad=True), torch.zeros(6, requires_grad=True)):
        time, times = d.classify_times(t, 6)
        assert time is None and times is t
    assert d.classify_times(torch.zeros(0, 1, requires_grad=True), 0)[1] is not None


def test_nan_rows_are_per_row():
    t = torch.tensor([float("nan"), 0.0, 0.0])
    assert d.classify_times(t, 3) == (None, t)


@pytest.mark.parametrize("t", [torch.linspace(-1, 1, 7), torch.linspace(-1, 1, 5).reshape(5, 1),
                               torch.full((7,), 0.1, requires_grad=True), torch.zeros(0, requires_grad=True)])
def test_other_element_counts_are_refused(t):
    with pytest.raises(ValueError, match="times_sel"):
        d.classify_times(t, 6)


def test_one_host_sync_for_a_tensor_of_equal_rows(monkeypatch):
    """the uniformity test reads the tensor back once, like the .item() of the one-time path"""
    calls = []
    orig = torch.Tensor.tolist

    def counted(self):
        calls.append(1)
        return orig(self)
    monkeypatch.setattr(torch.Tensor, "tolist", counted)
    monkeypatch.setattr(torch.Tensor, "item", lambda self: (_ for _ in ()).throw(AssertionError("item")))
    d.classify_times(torch.full((9, 1), 0.2), 9)
    d.classify_times(torch.linspace(0, 1, 9), 9)
    assert len(calls) == 2
