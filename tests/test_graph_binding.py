"""The key binding CapturedInference.Run derives from its inputs (he.py graph_binding): recorded input j's key slot is bound to the slot of
the input that takes its place; positions no input was recorded in keep their slot; one recorded slot bound to two slots is refused."""
import pytest

from cryptonets_b200.he import graph_binding


def test_each_recorded_slot_takes_its_inputs_slot():
    assert graph_binding([0], [0, 0, 0], [4, 4, 4]) == [4]
    assert graph_binding([1, 2, 3], [1, 2, 3], [3, 1, 2]) == [3, 1, 2]  # a permutation of the recorded clients
    assert graph_binding([1, 2, 3], [1, 2, 3], [5, 5, 6]) == [5, 5, 6]  # one client in two positions
    assert graph_binding([1, 2], [1, 2], [1, 2]) == [1, 2]  # the recording's own binding


def test_positions_without_an_input_keep_their_slot():
    assert graph_binding([0, 2, 7], [2], [9]) == [0, 9, 7]
    assert graph_binding([], [3], [4]) == []


def test_one_recorded_slot_bound_to_two_slots_is_refused():
    with pytest.raises(Exception, match="recorded key slot 2 to two key slots"):
        graph_binding([2], [2, 2], [5, 6])
