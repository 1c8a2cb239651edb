"""CPU: how torch.use_deterministic_algorithms selects the library's deterministic mode.

The library loads without a GPU and its switch (ub200_set_deterministic) is host state, so the policy of
uniter_b200._lib.select_mode / library_mode, and the autograd decorators that carry a forward's mode to
its backward, are checked here without launching anything.
"""
import warnings

import pytest
import torch

from uniter_b200 import _lib


@pytest.fixture
def flags():
    """Saves and restores torch's determinism flags and the library's switch."""
    lib = _lib.load()
    saved = (torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled())
    switch = lib.ub200_deterministic()

    def set_flags(on, warn_only=False):
        torch.use_deterministic_algorithms(on, warn_only=warn_only)
    yield set_flags
    torch.use_deterministic_algorithms(saved[0], warn_only=saved[1])
    lib.ub200_set_deterministic(switch)


@pytest.fixture
def switch_calls(monkeypatch):
    """Every value passed to ub200_set_deterministic, in order (the calls still reach the library)."""
    lib = _lib.load()
    real = lib.ub200_set_deterministic
    calls = []

    def spy(v):
        calls.append(v)
        return real(v)
    monkeypatch.setattr(lib, "ub200_set_deterministic", spy)
    return calls


@pytest.mark.parametrize("on,warn_only,want", [(False, False, None), (False, True, None),
                                               (True, False, 1), (True, True, 1)])
def test_each_combination_of_torch_flags_selects_the_mode(flags, on, warn_only, want):
    flags(on, warn_only)
    assert _lib.select_mode() == want
    assert _lib.select_mode(max_seqlen=128) == want          # the longest fixed-order attention backward
    assert _lib.select_mode(max_seqlen=64) == want


def test_a_long_attention_backward_is_refused_under_the_flag(flags):
    flags(True)
    with pytest.raises(RuntimeError, match=r"max_seqlen 129 > 128.*deterministic"):
        _lib.select_mode(max_seqlen=129)


def test_warn_only_runs_a_long_attention_backward_in_the_default_mode(flags):
    flags(True, warn_only=True)
    with pytest.warns(UserWarning, match=r"max_seqlen 512 > 128"):
        assert _lib.select_mode(max_seqlen=512) == 0


def test_a_long_attention_backward_is_left_alone_without_the_flag(flags):
    flags(False)
    with warnings.catch_warnings():
        warnings.simplefilter("error")
        assert _lib.select_mode(max_seqlen=512) is None


def test_library_mode_restores_the_previous_value(flags, switch_calls):
    lib = _lib.load()
    lib.ub200_set_deterministic(0)
    with _lib.library_mode(1):
        assert lib.ub200_deterministic() == 1
        assert _lib.select_mode() == 1                    # the enclosing scope decides, not torch's flags
        with _lib.library_mode(0):
            assert lib.ub200_deterministic() == 0
            assert _lib.select_mode(max_seqlen=512) == 0  # no second decision inside a default-mode scope
        assert lib.ub200_deterministic() == 1
    assert lib.ub200_deterministic() == 0
    lib.ub200_set_deterministic(1)                         # a C caller's setting survives a scope too
    with pytest.raises(ValueError):
        with _lib.library_mode(0):
            raise ValueError()
    assert lib.ub200_deterministic() == 1
    assert switch_calls == [0, 1, 0, 1, 0, 1, 0, 1]


def test_without_the_flag_the_switch_is_never_touched(flags, switch_calls):
    lib = _lib.load()
    flags(False)
    for c_value in (0, 1):                    # whatever a C caller set stays in force
        lib.ub200_set_deterministic(c_value)
        del switch_calls[:]
        with _lib.library_mode(_lib.select_mode(max_seqlen=512)):
            assert lib.ub200_deterministic() == c_value
        assert lib.ub200_deterministic() == c_value
        assert switch_calls == []


class _Probe(torch.autograd.Function):
    """Records the library's switch in its forward and backward (CPU tensors: nothing is launched)."""
    seen = []

    @staticmethod
    @_lib.forward_in_mode(lambda ctx, x, seqlen: seqlen)
    def forward(ctx, x, seqlen):
        _Probe.seen.append(("fwd", _lib.load().ub200_deterministic()))
        return x * 2

    @staticmethod
    @_lib.backward_in_mode
    def backward(ctx, g):
        _Probe.seen.append(("bwd", _lib.load().ub200_deterministic(), _lib.select_mode()))
        return g * 2, None


def _probe(seqlen=None):
    _Probe.seen = []
    x = torch.ones(3, requires_grad=True)
    return _Probe.apply(x, seqlen).sum()


def test_the_backward_runs_in_the_mode_of_its_forward(flags):
    lib = _lib.load()
    lib.ub200_set_deterministic(0)
    flags(True)
    y = _probe()
    flags(False)                             # switched off between forward and backward
    y.backward()
    assert _Probe.seen == [("fwd", 1), ("bwd", 1, 1)]
    assert lib.ub200_deterministic() == 0
    y = _probe()
    flags(True)                              # and on
    y.backward()
    assert _Probe.seen == [("fwd", 0), ("bwd", 0, None)]
    assert lib.ub200_deterministic() == 0


def test_a_long_forward_raises_or_runs_its_backward_in_the_default_mode(flags):
    lib = _lib.load()
    lib.ub200_set_deterministic(0)
    flags(True)
    with pytest.raises(RuntimeError, match="max_seqlen 200"):
        _probe(200)
    assert _Probe.seen == []                 # refused before any library work
    flags(True, warn_only=True)
    with pytest.warns(UserWarning, match="max_seqlen 200"):
        y = _probe(200)
    y.backward()
    assert _Probe.seen == [("fwd", 0), ("bwd", 0, 0)]
    y = _probe(128)
    y.backward()
    assert _Probe.seen == [("fwd", 1), ("bwd", 1, 1)]
    assert lib.ub200_deterministic() == 0
