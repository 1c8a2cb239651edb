"""CPU: FusedAdamW gives every element of shared parameter storage exactly one owner (_owned_ranges).

UniterForImageTextRetrieval.init_output() makes rank_output.weight / .bias views of row 1 of
itm_output.weight / .bias.  Both are parameters with gradients, so without a single owner two segments
of one adamw_kernel launch would write the same model addresses, in an order that varies from run to run.
"""
import pytest
import torch

from uniter_b200.optim import _owned_ranges


def test_disjoint_parameters_own_all_of_their_storage():
    a, b = torch.zeros(6, 4), torch.zeros(3)
    assert _owned_ranges([a, b]) == [[(0, 24)], [(0, 3)]]


def test_a_view_owns_its_rows_and_the_container_keeps_the_rest():
    from uniter_b200.heads import UniterForImageTextRetrieval
    from tests import util
    mod = UniterForImageTextRetrieval(util.tiny_config(), 64)
    mod.init_output()
    H = mod.itm_output.weight.size(1)
    params = [mod.itm_output.weight, mod.itm_output.bias, mod.rank_output.weight, mod.rank_output.bias]
    assert _owned_ranges(params) == [[(0, H)], [(0, 1)], [(0, H)], [(0, 1)]]
    assert _owned_ranges(params[::-1]) == [[(0, 1)], [(0, H)], [(0, 1)], [(0, H)]]


def test_nested_and_repeated_views():
    base = torch.zeros(10, 4)
    mid, inner = base[2:8], base[3:5]
    same = base[2:8]
    assert _owned_ranges([base, mid, inner]) == [[(0, 8), (32, 40)], [(0, 4), (12, 24)], [(0, 8)]]
    # identical ranges: the first listed owns them
    assert _owned_ranges([mid, same]) == [[(0, 24)], []]


def test_partial_overlap_is_refused():
    base = torch.zeros(10, 4)
    with pytest.raises(RuntimeError, match="share storage in part"):
        _owned_ranges([base[0:5], base[3:8]])
