"""The grouped-search oracle on hand-built cases: pins the semantics of search_groups independently of the GPU."""
from groups_oracle import group_search


def test_groups_ranked_by_best_row_and_truncated():
    scores = [0.9, 0.8, 0.7, 0.6, 0.5, 0.4]
    groups = ["a", "b", "a", "c", "a", "b"]
    assert group_search(scores, groups, 2, 2) == [("a", [(0, 0.9), (2, 0.7)]), ("b", [(1, 0.8), (5, 0.4)])]
    assert group_search(scores, groups, 10, 1) == [("a", [(0, 0.9)]), ("b", [(1, 0.8)]), ("c", [(3, 0.6)])]


def test_rows_without_a_group_are_never_returned():
    assert group_search([1.0, 0.5, 0.2], [None, "x", None], 5, 5) == [("x", [(1, 0.5)])]
    assert group_search([1.0], [None], 3, 3) == []


def test_ties_break_by_ascending_row():
    assert group_search([0.5, 0.5, 0.5], ["b", "a", "b"], 2, 2) == [("b", [(0, 0.5), (2, 0.5)]), ("a", [(1, 0.5)])]


def test_filter_restricts_both_choice_and_fill():
    scores = [0.9, 0.8, 0.7, 0.6]
    groups = ["a", "b", "a", "b"]
    assert group_search(scores, groups, 1, 2, rows=[1, 2, 3]) == [("b", [(1, 0.8), (3, 0.6)])]


def test_euclid_ranks_ascending():
    assert group_search([3.0, 1.0, 2.0], ["a", "b", "a"], 1, 2, ascending=True) == [("b", [(1, 1.0)])]


def test_typed_groups_stay_apart():
    groups = [("bool", True), ("int", 1), ("bool", True)]
    out = group_search([0.3, 0.2, 0.1], groups, 5, 5)
    assert out == [(("bool", True), [(0, 0.3), (2, 0.1)]), (("int", 1), [(1, 0.2)])]
