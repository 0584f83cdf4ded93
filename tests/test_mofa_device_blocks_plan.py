"""CPU: how the general mofa() path cuts a device-resident view into (view, group) blocks -- a zero-copy slice for an
ascending run of the view's rows without a feature mask, a gather otherwise -- and that a multi-process call of the
general path is still refused."""
from types import SimpleNamespace

import numpy as np
import pytest
import scipy.sparse as sp
import torch

from muon_b200 import _device, _dist, _mofa
from muon_b200._containers import SimpleAnnData, SimpleMuData


def _view(ad, dtype=torch.float32):
    """what _block_kind reads of a device view: its height and its value dtype"""
    return SimpleNamespace(shape=ad.shape, data=torch.empty(0, dtype=dtype))


def _plan(md, use_obs=None, groups_label=None, col_mask=None):
    """the block kind of every (view, group) and the rows it selects, as the general path computes them"""
    obs_all = np.asarray(md.obs_names).astype(str)
    common = np.intersect1d(*[np.asarray(a.obs_names) for a in md.mod.values()])
    cells, gid, names, ranges = _mofa._cell_layout(md, obs_all, common, use_obs, groups_label)
    pos_of = {c: i for i, c in enumerate(cells)}
    out = {}
    for m, ad in md.mod.items():
        per_g, _ = _mofa._view_rows(np.asarray(ad.obs_names).astype(str), pos_of, ranges)
        out[m] = [(_mofa._block_kind(_view(ad), rows, col_mask), rows.tolist()) for rows, _ in per_g]
    return names, ranges, out


def _md(n, obs_a=None, obs_b=None):
    names = [f"c{i}" for i in range(n)]
    obs_a = names if obs_a is None else obs_a
    obs_b = names if obs_b is None else obs_b
    a = SimpleAnnData(sp.random(len(obs_a), 5, density=0.5, format="csr", dtype=np.float32), obs=obs_a)
    b = SimpleAnnData(sp.random(len(obs_b), 4, density=0.5, format="csr", dtype=np.float32), obs=obs_b)
    return SimpleMuData({"a": a, "b": b})


def test_contiguous_groups_are_slices():
    md = _md(10)
    md.obs["grp"] = np.array(["x"] * 4 + ["y"] * 6)
    names, ranges, plan = _plan(md, groups_label="grp")
    assert names == ["x", "y"] and ranges == [(0, 4), (4, 10)]
    assert plan["a"] == [("slice", [0, 1, 2, 3]), ("slice", [4, 5, 6, 7, 8, 9])]
    # a feature mask turns every block into a gather (the mask is fused into it, not applied as a copy first)
    _, _, plan = _plan(md, groups_label="grp", col_mask=np.array([True, False, True, True, True]))
    assert [k for k, _ in plan["a"]] == ["gather", "gather"]


def test_interleaved_groups_are_gathers():
    md = _md(8)
    md.obs["grp"] = np.array(["x", "y"] * 4)
    names, ranges, plan = _plan(md, groups_label="grp")
    assert ranges == [(0, 4), (4, 8)]
    assert plan["a"] == [("gather", [0, 2, 4, 6]), ("gather", [1, 3, 5, 7])]
    # every view row lands in exactly one block: the gathers together copy the view once
    rows = sorted(r for _, rr in plan["b"] for r in rr)
    assert rows == list(range(8))


def test_union_with_missing_cells():
    names = [f"c{i}" for i in range(10)]
    md = _md(10, obs_a=names[:7], obs_b=names[3:])
    md.obs["grp"] = np.array(["x"] * 5 + ["y"] * 5)
    _, ranges, plan = _plan(md, use_obs="union", groups_label="grp")
    assert ranges == [(0, 5), (5, 10)]
    # view a holds c0..c6: rows 0..4 in x, 5..6 in y -- both ascending runs of its rows
    assert plan["a"] == [("slice", [0, 1, 2, 3, 4]), ("slice", [5, 6])]
    # view b holds c3..c9: c3, c4 in x (its rows 0, 1), c5..c9 in y (rows 2..6)
    assert plan["b"] == [("slice", [0, 1]), ("slice", [2, 3, 4, 5, 6])]
    # one group, the view's rows in a different order than the cells: gathers
    md2 = _md(6, obs_a=[f"c{i}" for i in range(6)], obs_b=[f"c{i}" for i in (5, 4, 3, 2, 1, 0)])
    _, _, plan2 = _plan(md2)
    assert plan2["a"] == [("slice", list(range(6)))]
    assert plan2["b"] == [("gather", [5, 4, 3, 2, 1, 0])]


def test_intersection_drops_cells():
    names = [f"c{i}" for i in range(10)]
    md = _md(10, obs_a=names[:8], obs_b=names[2:])
    md.obs["grp"] = np.array(["x", "y"] * 5)
    _, ranges, plan = _plan(md, use_obs="intersection", groups_label="grp")
    # c2..c7 are in both views; grouped x = c2, c4, c6 and y = c3, c5, c7
    assert ranges == [(0, 3), (3, 6)]
    assert plan["a"] == [("gather", [2, 4, 6]), ("gather", [3, 5, 7])]
    assert plan["b"] == [("gather", [0, 2, 4]), ("gather", [1, 3, 5])]
    # no groups: the common cells are one ascending run of each view's rows
    _, _, plan1 = _plan(md, use_obs="intersection")
    assert plan1["a"] == [("slice", [2, 3, 4, 5, 6, 7])]
    assert plan1["b"] == [("slice", [0, 1, 2, 3, 4, 5])]


def test_empty_block_is_a_slice():
    md = _md(6)
    md.obs["grp"] = np.array(["x"] * 6)
    names = [f"c{i}" for i in range(6)]
    md2 = _md(6, obs_a=names[:3], obs_b=names)
    md2.obs["grp"] = np.array(["x"] * 3 + ["y"] * 3)
    _, _, plan = _plan(md2, use_obs="union", groups_label="grp")
    assert plan["a"] == [("slice", [0, 1, 2]), ("slice", [])]


def _shard(ad, row0=0, n_total=None):
    """a device view of ad's shape that describes a cell shard (no entries; host tensors)"""
    n, d = ad.shape
    return _device.DeviceCSR(torch.zeros(n + 1, dtype=torch.int64), torch.empty(0, dtype=torch.int32),
                             torch.empty(0, dtype=torch.float32), (n, d), row0, n_total)


def test_identity_layout_takes_the_shard_of_the_first_device_view():
    """one group, no use_obs: every view's rows are None (all of them, in order, no names matched), and the initial
    factors' window and the group's cell count are the first DeviceCSR view's row0 / n_total"""
    md = _md(6)
    a, b = md.mod["a"], md.mod["b"]
    obs_all = np.asarray(md.obs_names).astype(str)
    host = sp.random(6, 4, density=0.5, format="csr")
    for Xs, window in (([_shard(a, 200, 1000), _shard(b)], (200, 1000)),
                       ([host, _shard(b, 40, 90)], (40, 90)),
                       ([host, host], (0, 6))):
        rows, names, ranges, totals, win, cells = _mofa._layout(md, Xs, obs_all, None, None, None, identity=True)
        assert rows == [[(None, (0, 6))], [(None, (0, 6))]]
        assert names == ["group1"] and ranges == [(0, 6)] and cells is None
        assert win == window and totals == [window[1]]
    # any other layout: the window is the N selected cells, whatever shard a view describes
    names6 = [f"c{i}" for i in range(6)]
    md2 = _md(6, obs_a=names6[:4], obs_b=names6[2:])
    md2.obs["grp"] = np.array(["x", "y"] * 3)
    obs_all = np.asarray(md2.obs_names).astype(str)
    Xs = [_shard(md2.mod["a"], 200, 1000), _shard(md2.mod["b"])]
    common = np.intersect1d(names6[:4], names6[2:])
    for use_obs, n in (("union", 6), ("intersection", 2)):
        rows, _, ranges, totals, win, (cells, cls) = _mofa._layout(md2, Xs, obs_all, common, use_obs, "grp",
                                                                   identity=False)
        assert win == (0, n) and sum(totals) == n and ranges[-1][1] == n
        # every factor-matrix row (cells ordered by group), its group and the views it is observed in
        want = [0, 2, 4, 1, 3, 5] if use_obs == "union" else [2, 3]
        assert cells.tolist() == [f"c{p}" for p in want]
        assert cls.tolist() == [((p % 2) << 2) | (p < 4) | ((p >= 2) << 1) for p in want]
    # a block whose cells are one run of the factor matrix is a row range, any other one a list of rows
    rows, *_ = _mofa._layout(md2, Xs, obs_all, common, "intersection", "grp", identity=False)
    assert [z for _, z in rows[0]] == [(0, 1), (1, 2)]
    rows, *_ = _mofa._layout(md2, Xs, obs_all, common, "union", "grp", identity=False)
    assert [z.tolist() for _, z in rows[0]] == [[0, 1], [3, 4]]


def test_distributed_general_path_is_refused(monkeypatch):
    md = _md(6)
    md.obs["grp"] = np.array(["x", "y"] * 3)
    monkeypatch.setattr(_dist, "is_distributed", lambda: True)
    with pytest.raises(NotImplementedError, match="single process"):
        _mofa.mofa(md, groups_label="grp", use_var=None)
    with pytest.raises(NotImplementedError, match="single process"):
        _mofa.mofa(_md(6), scale_groups=True, use_var=None)


def test_kind_follows_the_selection_rule_and_records_conversion():
    """_block_kind applies csr_select's own slice-or-gather rule; float64 views record their float32 copy"""
    md = _md(6)
    ad = md.mod["a"]
    mask = np.array([True, False, True, True, True])
    for rows in (None, np.arange(2, 5), np.array([], dtype=np.int64), np.array([3, 1]), np.array([1, 1])):
        for cm in (None, mask):
            want = "slice" if _device.select_is_view(rows, cm, 6) else "gather"
            assert _mofa._block_kind(_view(ad), rows, cm) == want
            assert _mofa._block_kind(_view(ad, torch.float64), rows, cm) == "convert+" + want
    assert _device.select_is_view(None, None, 6) and _device.select_is_view(np.arange(2, 5), None, 6)
    assert not _device.select_is_view(np.array([3, 1]), None, 6) and not _device.select_is_view(None, mask, 6)
