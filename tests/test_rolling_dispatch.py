"""CPU pin of the rolling-window and spell launch plans (launch_plan.cuh, through the host build of
tests/dispatch_host_build.py): a table naming every kernel instance the dispatch can pick, and the coverage of
tests/test_gpu_rolling_paths.py measured against it."""
import types

import pytest

import dispatch_host_build as H
from dispatch_host_build import MAX, MEAN, MIN, SUM, Unsupported

D = types.SimpleNamespace(spell_kernel=H.spell_instance, rolling_kernel=H.rolling_instance, slides=H.instance_slides,
                          can_stream4=H.can_stream4, INSTANCES=H.INSTANCES, SPELL_SUMW=H.SPELL_SUMW,
                          ROLLING_SUMW=H.ROLLING_SUMW, SLIDING=H.SLIDING)

RL = {"max": 0, "min": 1, "sum": 2, "count": 3, "mean": 4, "std": 5}
STAT = {"sum": 0, "mean": 1, "min": 2, "max": 3, "std": 4, "var": 5, "count": 6}
# spell_sumw_kernel's RED: MAX / SUM / COUNT keep their running form, the other reducers share kRunAny (-1)
SPELL_RED = {"max": 0, "sum": 2, "count": 3, "min": -1, "mean": -1, "std": -1}
ROLL_MODE = {"max": 0, "min": 1, "sum": 2, "mean": 2, "std": 2, "var": 2, "count": 2}


def _spell_table():
    rows = []
    for w in range(2, 9):
        for red, code in SPELL_RED.items():
            for before, after in ((True, "false"), (False, "true")):
                for wstat in (SUM, MEAN):
                    rows.append(((24, 24, w, wstat, RL[red], before, True), f"spell_sumw<{w}, {code}, {after}>", False))
    rows += [
        ((24, 24, 1, SUM, RL["count"], True, True), "spell_runstat4<false>", True),
        ((24, 24, 9, SUM, RL["count"], False, True), "spell_runstat4<true>", True),
        ((2052, 2056, 80, MEAN, RL["max"], True, True), "spell_runstat4<false>", True),     # the ring at its cap
        ((24, 24, 81, SUM, RL["max"], True, True), "spell_runstat", True),                  # 162 kB: over it
        ((24, 24, 3, MIN, RL["max"], True, True), "spell_runstat4<false>", False),
        ((24, 24, 80, MAX, RL["max"], False, True), "spell_runstat4<true>", False),
        ((24, 25, 3, SUM, RL["max"], True, True), "spell_runstat", False),                  # offset slice
        ((24, 25, 7, SUM, RL["max"], True, True), "spell_runstat", True),                   # slides above w = 6
        ((24, 28, 5, SUM, RL["sum"], False, False), "spell_runstat", False),                # base off 16 bytes
        ((3, 3, 5, SUM, RL["sum"], True, True), "spell_runstat", False),                    # C % 4 != 0
        ((1028, 1032, 5, SUM, RL["sum"], True, True), "spell_sumw<5, 2, false>", False),    # band view
    ]
    return rows


def _rolling_table():
    rows = []
    for w in range(2, 9):
        for stat, mode in ROLL_MODE.items():
            for wstat in (SUM, MEAN):
                rows.append(((24, 24, w, wstat, STAT[stat], False, True), f"rolling_sumw<{w}, {mode}>", False))
    rows += [
        ((24, 24, 1, SUM, STAT["min"], False, True), "rolling_period_reduce4", True),
        ((24, 24, 9, MEAN, STAT["max"], True, True), "rolling_period_reduce4", True),
        ((24, 24, 80, SUM, STAT["sum"], False, True), "rolling_period_reduce4", True),
        ((24, 24, 81, SUM, STAT["sum"], True, True), "rolling_period_reduce", True),
        ((24, 24, 5, MAX, STAT["sum"], True, True), "rolling_period_reduce4", False),
        ((24, 25, 3, SUM, STAT["sum"], False, True), "rolling_period_reduce", True),
        ((3, 3, 2, MIN, STAT["max"], False, True), "rolling_period_reduce", False),
        ((24, 24, 3, SUM, STAT["max"], False, False), "rolling_period_reduce", True),
    ]
    return rows


@pytest.mark.parametrize("args,kernel,slides", _spell_table())
def test_spell_dispatch(args, kernel, slides):
    C, ldx, w, wstat, red, before, aligned = args
    assert D.spell_kernel(C, ldx, w, wstat, red, before, aligned_x=aligned) == kernel
    assert D.slides(kernel, w, wstat) is slides


@pytest.mark.parametrize("args,kernel,slides", _rolling_table())
def test_rolling_dispatch(args, kernel, slides):
    C, ldx, w, wstat, stat, center, aligned = args
    assert D.rolling_kernel(C, ldx, w, wstat, stat, center, aligned_x=aligned) == kernel
    assert D.slides(kernel, w, wstat) is slides


def test_tables_name_every_instance():
    named = {k for _, k, _ in _spell_table() + _rolling_table()} | {"spell_mask"}
    assert named == set(D.INSTANCES)
    assert len(D.SPELL_SUMW) == 56 and len(D.ROLLING_SUMW) == 21 and len(set(D.INSTANCES)) == len(D.INSTANCES)


def test_ring_cap_and_even_centre():
    assert D.can_stream4(24, 24, 80) and not D.can_stream4(24, 24, 81)
    assert not D.can_stream4(24, 26, 3) and not D.can_stream4(22, 24, 3) and not D.can_stream4(24, 24, 3, False)
    with pytest.raises(Unsupported):
        D.rolling_kernel(24, 24, 4, SUM, STAT["sum"], center=True)
    assert D.slides("spell_mask", 6, SUM) is False and D.slides("spell_mask", 7, MEAN) is True
    assert D.slides("spell_mask", 12, MAX) is False


def test_gpu_cases_reach_every_instance():
    """tests/test_gpu_rolling_paths.py launches every instance of the dispatch, and every sliding path with
    hostile data (an infinity or a huge value early in a period)."""
    import test_gpu_rolling_paths as G
    reached = G.expected_instances()
    assert reached == set(D.INSTANCES), sorted(set(D.INSTANCES) - reached)
    assert G.hostile_sliding_instances() == D.SLIDING
