"""GPU: the peak-ranking kernels (csrc/rank.cu) against exact references at every size class the host routes a peak
to, at the class edges, in both precisions, and at the limits of the C ABI -- workspace slices reused by many long
rows, 1 to 1024 tested groups, 2 642 244 ranked cells with tie blocks past 2^21 cells -- plus the score kernel's
p-values against mpmath over the whole (t, df) range, and the benchmark's matrix sampled peak by peak.

Where a path must be pinned, ``mub_rank_stats_f32/_f64`` and ``mub_rank_score`` are called through the C ABI, so that
the host's routing cannot hide a failure; ``_rank.peak_stats`` / ``rank_peaks_groups`` are called where the routing
itself is under test.  Counts, rank sums (half-integers below 2^53) and tie terms (float of the exact integer) must
equal the float64 oracle exactly."""
import math

import numpy as np
import pandas as pd
import pytest
import scipy.sparse as sp
import torch

from muon_b200 import _lib, _rank
from muon_b200._lib import (RANK_OVERESTIM_VAR, RANK_VS_GROUP, RANK_WILCOXON, MuonB200Error, call, load, ptr,
                            stream_ptr)
from oracle import rank_ref as R

pytestmark = pytest.mark.gpu

EPS = np.finfo(np.float64).eps


# ---- helpers ---------------------------------------------------------------------------------------------------------
def _plan(labels, n_cat, groups="all", reference="rest"):
    cat = pd.Categorical.from_codes(np.asarray(labels, dtype=np.int64), categories=[str(i) for i in range(n_cat)])
    return _rank.Plan(pd.Series(cat), groups, reference)


def _routed(T, plan, peaks=None, tie_correct=True):
    """peak_stats over the peaks of T (peaks x cells, host CSR): the host picks every row's size class."""
    A = _rank.device_matrix(sp.csr_matrix(T.T))
    peaks = np.arange(T.shape[0]) if peaks is None else peaks
    st, long_share, flags = _rank.peak_stats(A, plan, peaks, wilcoxon=True, tie_correct=tie_correct)
    torch.cuda.synchronize()
    return st, long_share, flags


def _abi(T, plan, flags, cap, slices=4, rows=None):
    """mub_rank_stats_* over rows of T with one explicit cap (a short class, or the long path when cap exceeds the
    shared capacity; then ``slices`` workspace slices)."""
    dev = torch.device("cuda", 0)
    vb = T.data.dtype.itemsize
    indptr = torch.from_numpy(T.indptr.astype(np.int64)).to(dev)
    cells = torch.from_numpy(T.indices.astype(np.int32)).to(dev)
    vals = torch.from_numpy(T.data).to(dev)
    rows = np.arange(T.shape[0]) if rows is None else np.asarray(rows)
    r = torch.from_numpy(rows.astype(np.int32)).to(dev)
    code, sizes = torch.from_numpy(plan.code).to(dev), torch.from_numpy(plan.sizes).to(dev)
    K = len(plan.tested) + 1
    out = torch.full((5, K, len(rows)), float("nan"), dtype=torch.float64, device=dev)
    ws, ws_bytes = None, 0
    if cap > load().mub_rank_shared_capacity(vb):
        ws_bytes = slices * int(load().mub_rank_workspace_slice_bytes(vb, cap))
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    call("mub_rank_stats_f64" if vb == 8 else "mub_rank_stats_f32", ptr(indptr), ptr(cells), ptr(vals), ptr(code),
         ptr(r), ptr(r), len(rows), len(rows), K, ptr(sizes), plan.n_ranked, flags, cap, ptr(ws), ws_bytes, ptr(out),
         stream_ptr())
    torch.cuda.synchronize()
    return out


def _same(a, b):
    """Identical bits (a sum over +inf and -inf is NaN, which torch.equal never calls equal)."""
    return a.shape == b.shape and torch.equal(a.view(torch.int64), b.view(torch.int64))


def _long_cap(T, vb):
    """A cap that sends every row of T through the global-memory sort."""
    longest = int(np.diff(T.indptr).max())
    return max(2 * int(load().mub_rank_shared_capacity(vb)), 1 << max(1, (longest - 1).bit_length()))


def _oracle(T, plan, labels, peaks=None):
    """group_stats of the float64 oracle on the columns ``peaks`` of the cells x peaks matrix T^T."""
    peaks = np.arange(T.shape[0]) if peaks is None else np.asarray(peaks)
    dense = np.ascontiguousarray(T[peaks].toarray().T)
    groups = plan.tested + ([plan.reference] if plan.reference is not None else [])
    lab = np.asarray(labels)
    masks = np.stack([lab == int(g) for g in groups])
    ref = len(plan.tested) if plan.reference is not None else None
    return R.group_stats(dense, masks, ref, tie_correct=True)


def _check(st, want, plan, rows=None, sums=True, mag=None):
    """Exact counts, rank sums and tie terms of the tested groups (and the reference's count); sums and sums of squares
    to rtol 1e-12, or the sums to 1e-12 of ``mag`` [K][peaks], the sums of magnitudes, where they may cancel."""
    st = st.cpu().numpy() if torch.is_tensor(st) else st
    G = len(plan.tested)
    rows = slice(None) if rows is None else rows
    np.testing.assert_array_equal(st[0, :G][:, rows], want["cnt"][:G][:, rows])
    np.testing.assert_array_equal(st[3, :G][:, rows], want["ranksum"][:G][:, rows])
    np.testing.assert_array_equal(st[4, :G][:, rows], want["tie"][:G][:, rows])
    if plan.reference is not None:
        np.testing.assert_array_equal(st[0, G][rows], want["cnt"][G][rows])
    if sums:
        K = G + (plan.reference is not None)
        for q, key in ((1, "sum"), (2, "sumsq")):
            got, ref = st[q, :K][:, rows], want[key][:K][:, rows]
            if q == 1 and mag is not None:
                assert np.all(np.abs(got - ref) <= 1e-12 * mag[:K][:, rows])
            else:
                np.testing.assert_allclose(got, ref, rtol=1e-12, atol=1e-300)


def _magnitudes(T, plan, labels):
    """[K][peaks] sums of |x| over each group's stored entries of each peak."""
    groups = plan.tested + ([plan.reference] if plan.reference is not None else [])
    onehot = sp.csr_matrix(np.stack([np.asarray(labels) == int(g) for g in groups]).T.astype(np.float64))
    return np.asarray((abs(T).astype(np.float64) @ onehot).T.todense())


def _z64(want, plan, n, tie_correct):
    """The Wilcoxon z of scanpy in float64 from the oracle's statistics."""
    G = len(plan.tested)
    ng = plan.sizes[:G].astype(np.float64)[:, None]
    N = n if plan.reference is None else ng + plan.sizes[G]
    T = 1.0 - want["tie"][:G] / (N**3 - N) if tie_correct else 1.0
    with np.errstate(invalid="ignore", divide="ignore"):
        z = (want["ranksum"][:G] - ng * (N + 1) / 2) / np.sqrt(T * ng * (N - ng) * (N + 1) / 12.0)
    z[np.isnan(z)] = 0
    return z


# ---- 1a: every size class, at its edges, in both precisions ----------------------------------------------------------
N_EDGE = 150_000
EDGE_SIZES = np.array([0.3, 0.2, 0.15, 0.12, 0.1, 0.08, 0.05])   # 7 categories of skewed sizes


def _edge_lengths(cap):
    return [0, 1, 2, 511, 512, 513, 2047, 2048, 2049, cap - 1, cap, cap + 1, 2 * cap, 2 * cap + 1, 8 * cap + 1]


def _edge_matrix(dtype, seed=0):
    """peaks x cells CSR whose rows have the stored lengths of _edge_lengths, in random cell order.  Stored but not
    ranked: explicit zeros and -0.0.  Dyadic values with many ties and negatives; rows of 2 cap or more hold a tie block
    longer than a chunk (cap entries), each spread over every group; from 16 entries on, subnormals and neighbours one
    ulp apart; odd rows ("wild") also +-max and +-inf, whose sums are not compared."""
    V = np.dtype(dtype)
    cap = int(load().mub_rank_shared_capacity(V.itemsize))
    rng = np.random.default_rng(seed)
    fi = np.finfo(V)
    sub = fi.smallest_subnormal if hasattr(fi, "smallest_subnormal") else np.nextafter(V.type(0), V.type(1))
    one = V.type(1)
    indptr, indices, data, wild = [0], [], [], []
    for i, L in enumerate(_edge_lengths(cap)):
        cells = rng.choice(N_EDGE, size=L, replace=False).astype(np.int32)
        v = (rng.integers(-12, 25, size=L) * 0.25).astype(V)          # k/4: 0 is an explicit stored zero
        v[rng.random(L) < 0.03] = V.type(-0.0)
        o = 0
        if L >= 2 * cap:
            v[:int(1.3 * cap)] = V.type(1.5)
            v[int(1.3 * cap):int(1.9 * cap)] = V.type(-0.75)
            o = int(1.9 * cap)
        if L >= 16:
            extra = [sub, -sub, 2 * sub, 3 * sub, one, np.nextafter(one, V.type(2)), np.nextafter(one, V.type(0)),
                     -np.nextafter(one, V.type(2))]
            if i % 2:
                extra += [fi.max, -fi.max, np.nextafter(fi.max, V.type(0)), V.type(np.inf), V.type(-np.inf), fi.max]
            v[o:o + len(extra)] = np.array(extra, dtype=V)
        wild.append(bool(i % 2) and L >= 16)
        v = v[rng.permutation(L)]
        indices.append(cells)
        data.append(v)
        indptr.append(indptr[-1] + L)
    T = sp.csr_matrix((np.concatenate(data), np.concatenate(indices), np.array(indptr, dtype=np.int64)),
                      shape=(len(indptr) - 1, N_EDGE))
    labels = rng.choice(len(EDGE_SIZES), size=N_EDGE, p=EDGE_SIZES)
    return T, labels, np.array(wild)


@pytest.fixture(scope="module", params=["float32", "float64"])
def edge_case(request):
    T, labels, wild = _edge_matrix(request.param)
    assert T.nnz == sum(_edge_lengths(int(load().mub_rank_shared_capacity(T.data.dtype.itemsize))))
    return T, labels, wild


@pytest.mark.parametrize("reference", ["rest", "5"])
def test_every_size_class_at_its_edges(edge_case, reference, cuda):
    """Each row routed to its class (512, 2048, full, long) equals the oracle exactly, and gives the same bits when
    forced through the global-memory sort; the scores with and without the tie correction equal float64 z."""
    T, labels, wild = edge_case
    vb = T.data.dtype.itemsize
    groups = "all" if reference == "rest" else ["0", "1", "2", "3", "4"]      # against "5": cells of "6" are unranked
    plan = _plan(labels, len(EDGE_SIZES), groups, reference)
    assert (plan.code == -1).any() == (reference != "rest")
    st, long_share, flags = _routed(T, plan)
    cap = int(load().mub_rank_shared_capacity(vb))
    lengths = np.diff(T.indptr)
    assert long_share == pytest.approx(lengths[lengths > cap].sum() / lengths.sum())
    want = _oracle(T, plan, labels)
    _check(st, want, plan, sums=False)
    _check(st, want, plan, rows=~wild, mag=_magnitudes(T, plan, labels))
    forced = _abi(T, plan, flags, _long_cap(T, vb), slices=3)
    assert _same(forced, st)
    for tie_correct in (False, True):
        st2, _, flags2 = _routed(T, plan, tie_correct=tie_correct)
        assert _same(st2, st)                      # the statistics do not depend on the correction
        scores = _rank.score(st2, plan, flags2, N_EDGE)[0].cpu().numpy()
        np.testing.assert_allclose(scores, _z64(want, plan, N_EDGE, tie_correct), rtol=1e-12, atol=1e-13)


def test_each_class_pinned_through_the_abi(edge_case, cuda):
    """Every row launched at every cap that holds it (512, 2048, the full class, the long path): identical bits."""
    T, labels, _ = edge_case
    vb = T.data.dtype.itemsize
    cap_shared = int(load().mub_rank_shared_capacity(vb))
    lengths = np.diff(T.indptr)
    for reference in ("rest", "5"):
        groups = "all" if reference == "rest" else ["0", "1", "2", "3", "4"]
        plan = _plan(labels, len(EDGE_SIZES), groups, reference)
        flags = RANK_WILCOXON | (RANK_VS_GROUP if plan.reference is not None else 0)
        base = _abi(T, plan, flags, _long_cap(T, vb))
        for cap in (512, 2048, cap_shared):
            rows = np.flatnonzero(lengths <= cap)
            got = _abi(T, plan, flags, cap, rows=rows)
            assert _same(got, base[:, :, torch.from_numpy(rows).cuda()].contiguous()), cap


# ---- 1b: workspace slices reused by many long rows -------------------------------------------------------------------
@pytest.mark.parametrize("dtype", ["float32", "float64"])
def test_workspace_reuse(dtype, monkeypatch, cuda):
    """48 long rows, longest first, then shortest, then longest again, through 1, 2 and 3 workspace slices: each CTA
    sorts many rows of different lengths in one slice.  Bit-identical to the default workspace and exact."""
    V = np.dtype(dtype)
    cap = int(load().mub_rank_shared_capacity(V.itemsize))
    rng = np.random.default_rng(11)
    n = 3 * cap + 4096
    lengths = [cap + 1 + abs(i - 24) * (2 * cap // 24) for i in range(48)]
    indptr = np.concatenate([[0], np.cumsum(lengths)]).astype(np.int64)
    cells = np.concatenate([rng.choice(n, size=L, replace=False) for L in lengths]).astype(np.int32)
    vals = (rng.integers(-6, 10, size=indptr[-1]) * 0.5).astype(V)
    T = sp.csr_matrix((vals, cells, indptr), shape=(len(lengths), n))
    labels = rng.integers(0, 4, size=n)
    for reference, groups in (("rest", "all"), ("3", ["0", "1"])):
        plan = _plan(labels, 4, groups, reference)
        default, share, _ = _routed(T, plan)
        assert share == 1.0
        _check(default, _oracle(T, plan, labels), plan)
        slice_bytes = int(load().mub_rank_workspace_slice_bytes(V.itemsize, 1 << (max(lengths) - 1).bit_length()))
        for slices in (1, 2, 3):
            monkeypatch.setattr(_rank, "LONG_WORKSPACE", slices * slice_bytes)
            st, _, _ = _routed(T, plan)
            assert _same(st, default), (reference, slices)
        monkeypatch.undo()


# ---- 1c: group counts ------------------------------------------------------------------------------------------------
N_GROUPS_CELLS = 24_000
N_CATS = 1100


def _groups_matrix(seed=3):
    """Rows of 0, 300 (512 class), 1500 (2048 class), 10 000 (full class) and 20 000 (long path) entries over 1100
    categories of about 22 cells each: with 1024 groups most groups have no entry in the short rows."""
    rng = np.random.default_rng(seed)
    lengths = [0, 300, 1500, 10_000, 20_000]
    indptr = np.concatenate([[0], np.cumsum(lengths)]).astype(np.int64)
    cells = np.concatenate([rng.choice(N_GROUPS_CELLS, size=L, replace=False) for L in lengths]).astype(np.int32)
    vals = rng.integers(-3, 6, size=indptr[-1]).astype(np.float32)
    labels = np.arange(N_GROUPS_CELLS) % N_CATS
    rng.shuffle(labels)
    return sp.csr_matrix((vals, cells, indptr), shape=(len(lengths), N_GROUPS_CELLS)), labels


@pytest.mark.parametrize("G", [1, 2, 1024])
@pytest.mark.parametrize("against", ["rest", "group"])
def test_group_counts(G, against, cuda):
    """1, 2 and RANK_MAX_GROUPS tested groups on every class; the rest holds most cells at G = 1, 2 (a tested subset),
    and at G = 1024 the fp32 full class launches with K = 1025 (~184 KB of shared memory)."""
    T, labels = _groups_matrix()
    groups = [str(g) for g in range(0, 2 * G, 2)] if G < 1024 else [str(g) for g in range(G)]
    reference = "rest" if against == "rest" else "1099"
    plan = _plan(labels, N_CATS, groups, reference)
    assert len(plan.tested) == G
    st, share, flags = _routed(T, plan)
    assert 0 < share < 1
    want = _oracle(T, plan, labels)
    _check(st, want, plan)
    if G == 1024:
        assert (st[0, :G, 1] == 0).sum().item() > 600      # groups with no entry in the 300-entry row
    scores = _rank.score(st, plan, flags, N_GROUPS_CELLS)[0].cpu().numpy()
    np.testing.assert_allclose(scores, _z64(want, plan, N_GROUPS_CELLS, True), rtol=1e-12, atol=1e-13)


def test_group_count_limits(cuda):
    """1025 tested groups are refused before any device work; K = 1026 is refused by the C ABI."""
    T, labels = _groups_matrix()
    with pytest.raises(NotImplementedError):
        _plan(labels, N_CATS, [str(g) for g in range(_lib.RANK_MAX_GROUPS + 1)])
    plan = _plan(labels, N_CATS, [str(g) for g in range(_lib.RANK_MAX_GROUPS)], "1099")
    assert len(plan.tested) + 1 == _lib.RANK_MAX_GROUPS + 1
    plan.tested = plan.tested + ["1098"]                 # K = 1026 handed straight to the C ABI
    with pytest.raises(MuonB200Error, match="groups"):
        _abi(T, plan, RANK_WILCOXON | RANK_VS_GROUP, 512, rows=[1])


# ---- 1d: the ranked-cell limit ---------------------------------------------------------------------------------------
def test_ranked_cell_limit(cuda):
    """2 642 244 ranked cells: one peak holds a stored tie block of 2 200 000 equal values, one leaves a zero block of
    about 2.6M cells, one mixes both.  Tie terms near 1.8e19 equal the exact integers rounded to float64, rank sums are
    exact.  One cell more is refused by peak_stats and by the C ABI."""
    n = _rank.RANKED_CELLS_LIMIT - 1
    rng = np.random.default_rng(7)
    labels = np.where(rng.random(n) < 0.85, 2, rng.integers(0, 2, size=n))      # "2": 85 % of the cells
    big = rng.choice(n, size=2_200_000, replace=False)
    few = rng.choice(n, size=5000, replace=False)
    mix = rng.choice(n, size=300_000, replace=False)
    rows = [(big, np.where(np.arange(big.size) < 2_150_000, 2.0, rng.integers(-2, 3, size=big.size))),
            (few, rng.integers(1, 4, size=few.size).astype(np.float64)),
            (mix, rng.integers(-1, 3, size=mix.size).astype(np.float64))]
    indptr = np.concatenate([[0], np.cumsum([c.size for c, _ in rows])]).astype(np.int64)
    T = sp.csr_matrix((np.concatenate([v for _, v in rows]).astype(np.float32),
                       np.concatenate([c for c, _ in rows]).astype(np.int32), indptr), shape=(3, n))
    for reference, groups in (("rest", "all"), ("2", ["0"])):
        plan = _plan(labels, 3, groups, reference)
        assert plan.n_ranked == n if reference == "rest" else plan.n_ranked < n
        st, share, _ = _routed(T, plan)
        assert share > 0.5
        want = _oracle(T, plan, labels)
        _check(st, want, plan)
        assert want["tie"][0].max() > 1e19 if reference == "rest" else want["tie"][0].max() > 5e18
    # one more ranked cell
    over = np.concatenate([labels, [0]])
    plan = _plan(over, 3)
    assert plan.n_ranked == _rank.RANKED_CELLS_LIMIT
    with pytest.raises(NotImplementedError):
        _routed(sp.csr_matrix((3, n + 1), dtype=np.float32), plan)
    with pytest.raises(MuonB200Error, match="ranked cells"):
        _abi(T, plan, RANK_WILCOXON, 512)


# ---- 1e: the score kernel --------------------------------------------------------------------------------------------
DF_GRID = [1, 1.5, 2, 3, 10, 39.99, 40, 40.01, 1e3, 1e5, 1e6, 2.6e6]


def _score(stats, sizes, n_total, flags, log_base=0.0):
    dev = torch.device("cuda", 0)
    st = torch.from_numpy(np.ascontiguousarray(stats)).to(dev)
    K, n_out = stats.shape[1], stats.shape[2]
    out = [torch.full((K - 1, n_out), float("nan"), dtype=torch.float64, device=dev) for _ in range(3)]
    pts = torch.zeros((K, n_out), dtype=torch.float64, device=dev)
    pts_rest = torch.zeros((K - 1, n_out), dtype=torch.float64, device=dev)
    g_n = torch.tensor(sizes, dtype=torch.int64, device=dev)
    call("mub_rank_score", ptr(st), K, n_out, ptr(g_n), n_total, flags, log_base, ptr(out[0]), ptr(out[1]),
         ptr(out[2]), ptr(pts), ptr(None if flags & RANK_VS_GROUP else pts_rest), stream_ptr())
    torch.cuda.synchronize()
    return [t.cpu().numpy() for t in out] + [pts.cpu().numpy(), pts_rest.cpu().numpy()]


def _round_bits(x, bits):
    if x == 0:
        return 0.0
    m, e = math.frexp(x)
    return math.ldexp(round(m * 2**bits), e - bits)


def _ttest_point(df, t):
    """(stats column of group 0 and group 1, n0, n1) whose Welch t and df are near (t, df) and whose variances come out
    of the kernel's (sum of squares / n - mean^2) without rounding that FMA contraction could change: the mean of group
    0 has 26 significant bits, its mean of squares 31, group 1 has mean 0.  Far tails of integer df use a group 0 of
    zero variance (then df = n1 - 1), which is the only way float64 moments reach |t| beyond ~1e4."""
    if abs(t) > 1e3:
        assert df == int(df)
        n0, n1 = 2, int(df) + 1
        m = math.copysign(_round_bits(math.sqrt(abs(t)), 26), t)      # m^2 and (m / t)^2 both in range
        vn2 = (m / t) ** 2
        return [1, m * n0, n0 * m * m], [1, 0.0, vn2 * n1 * (n1 - 1)], n0, n1
    N = math.ceil(df / 2) + 1                           # df(rho) = (1 + rho)^2 (N-1) / (1 + rho^2) on [N-1, 2(N-1)]
    lo, hi = 1.0, 1e12
    for _ in range(200):
        mid = math.sqrt(lo * hi)
        lo, hi = (mid, hi) if (1 + mid) ** 2 * (N - 1) / (1 + mid * mid) > df else (lo, mid)
    rho = lo
    vn1 = 2.0**-4
    m = _round_bits(t * math.sqrt(vn1 * (1 + rho)), 26)
    q0 = _round_bits(vn1 * N * (N - 1) / N + m * m, 31)
    return [1, m * N, q0 * N], [1, 0.0, rho * vn1 * N * (N - 1)], N, N


def _t_df(stats, n0, n1, overestim=False):
    """Welch's t and df from the statistics, in the kernel's float64 operations."""
    s = stats
    mg, mr = s[1, 0] / n0, s[1, 1] / n1
    vg = (s[2, 0] / n0 - mg * mg) * (n0 / (n0 - 1.0))
    vr = (s[2, 1] / n1 - mr * mr) * (n1 / (n1 - 1.0))
    n2 = n0 if overestim else n1
    a, b = vg / n0, vr / n2
    with np.errstate(invalid="ignore", divide="ignore"):
        df = (a + b) * (a + b) / (a * a / (n0 - 1.0) + b * b / (n2 - 1.0))
        t = (mg - mr) / np.sqrt(a + b)
    return t, np.where(np.isnan(df), 1.0, df)


def _p_ref(t, df):
    import mpmath as mp
    with mp.workdps(40):
        t, df = mp.mpf(float(t)), mp.mpf(float(df))
        if t == 0:
            return mp.mpf(1)
        return mp.betainc(df / 2, mp.mpf(1) / 2, 0, df / (df + t * t), regularized=True)


def _p_tol(p_ref):
    """1e-13, plus the conditioning of p on its argument: d ln p / d ln t ~ -2u with u ~ -ln p, so the half-ulp
    rounding of t^2 / df (or of |z| / sqrt 2) alone moves p by about eps * |ln p|, up to 1.5e-13 at p ~ 1e-300.
    scipy.stats.t.sf lands in the same band there (1.6e-13 at p ~ 1e-280, df = 1e6)."""
    return 1e-13 + 4 * EPS * max(0.0, -float(np.log(float(p_ref)))) if p_ref > 0 else 1e-13


def _t_grid(df):
    """|t| from 1e-12 up to where p falls below 1e-300 (about 40 points), and t = 0."""
    from scipy import stats as S
    hi = 1.0
    while S.t.logsf(hi, df) > math.log(0.5e-300):
        hi *= 2.0
    if df != int(df):
        hi = min(hi, 1e3)
    return [0.0] + list(np.geomspace(1e-12, 1e-1, 6)) + list(np.linspace(0.25, 5, 12)) + \
        list(np.geomspace(5.5, hi, 22))


def test_student_p_against_mpmath(cuda):
    """The two-sided t-test p over df in DF_GRID (the Stirling switch of ln B(a, 1/2) at df = 40; the large-a series
    from df = 600 on) and |t| from 1e-12 to where p < 1e-300, against mpmath at the kernel's own t and at df recomputed
    in float64 from the same statistics, so that rounding in t cannot count against the kernel.  The continued fraction
    alone loses about (df / 2) eps: 2e-12 at df = 1e5 and t ~ 2-3."""
    cols, meta = [], []
    for df in DF_GRID:
        for t in _t_grid(df):
            for sign in (1.0, -1.0):
                g, r, n0, n1 = _ttest_point(df, sign * t)
                cols.append((g, r))
                meta.append((n0, n1))
    # one launch per (n0, n1): group sizes are per launch
    by_n = {}
    for i, nn in enumerate(meta):
        by_n.setdefault(nn, []).append(i)
    worst, cache = 0.0, {}
    for vs_ref in (False, True):
        for (n0, n1), idx in by_n.items():
            stats = np.zeros((5, 2, len(idx)))
            for j, i in enumerate(idx):
                stats[:3, 0, j], stats[:3, 1, j] = cols[i]
            flags = RANK_VS_GROUP if vs_ref else 0
            scores, pvals, *_ = _score(stats, [n0, n1], n0 + n1, flags)
            t64, df64 = _t_df(stats, n0, n1)
            np.testing.assert_allclose(scores[0], t64, rtol=4 * EPS, atol=0)
            for j in range(len(idx)):
                key = (float(scores[0, j]), float(df64[j]))
                want = cache[key] if key in cache else cache.setdefault(key, _p_ref(*key))
                if want < 1e-300:
                    continue
                err = abs(pvals[0, j] - float(want)) / float(want)
                worst = max(worst, err / _p_tol(want))
                assert err <= _p_tol(want), (scores[0, j], df64[j], pvals[0, j], float(want), err)
    assert worst > 0


def test_student_p_huge_t_at_small_df(cuda):
    """df = 1 keeps p = 2 / (pi |t|) far above the smallest double even where t^2 overflows."""
    stats = np.zeros((5, 2, 3))
    for j, (m, sq) in enumerate(((2.0**500, 2.0**-100), (2.0**510, 2.0**-600), (2.0**511, 2.0**-890))):
        stats[:3, 0, j] = [1, 2 * m, 2 * m * m]          # group 0 (2 cells): mean m, variance 0
        stats[:3, 1, j] = [1, 0.0, sq]                   # group 1 (2 cells): mean 0, variance sq; df = 1
    scores, pvals, *_ = _score(stats, [2, 2], 4, RANK_VS_GROUP)
    assert np.all(scores[0] > 1e165) and np.all(scores[0] ** 2 == np.inf)
    for j in range(3):
        want = _p_ref(scores[0, j], 1.0)
        assert want > 1e-300 and abs(pvals[0, j] - float(want)) <= _p_tol(want) * float(want), j


def test_wilcoxon_p_against_mpmath(cuda):
    """p = erfc(|z| / sqrt 2) for |z| up to 38 (p ~ 3e-316), at the z the kernel returned."""
    import mpmath as mp
    z_want = np.concatenate([[0.0], np.geomspace(1e-10, 1, 8), np.linspace(1.5, 38, 40)])
    z_want = np.concatenate([z_want, -z_want[1:]])
    ng, nr = 4000, 6000
    N = ng + nr
    sd = math.sqrt(ng * nr * (N + 1) / 12.0)
    stats = np.zeros((5, 2, len(z_want)))
    stats[3, 0] = np.round((z_want * sd + ng * (N + 1) / 2) * 2) / 2      # half-integer rank sums
    for flags in (RANK_WILCOXON, RANK_WILCOXON | RANK_VS_GROUP):
        scores, pvals, *_ = _score(stats, [ng, nr], N, flags)
        np.testing.assert_allclose(scores[0], (stats[3, 0] - ng * (N + 1) / 2) / sd, rtol=1e-14, atol=1e-15)
        for z, p in zip(scores[0], pvals[0]):
            with mp.workdps(40):
                want = mp.erfc(abs(mp.mpf(float(z))) / mp.sqrt(2))
            if want < 1e-300:
                continue
            assert abs(p - float(want)) <= _p_tol(want) * float(want), (z, p, float(want))


def test_score_rules(cuda):
    """NaN df -> p from df = 1; zero variances: t = +-inf -> p = 0, t = NaN -> score 0 and p 1; the overestimated
    variance uses n_g for the other group; pts / pts_rest; log fold changes with log_base None, 2 and 10."""
    from scipy import stats as S
    # NaN df: both variances per cell 2^-565, (2^-564)^2 underflows to 0 -> df = 0 / 0; t = 2^-280 / 2^-282 = 4
    m = 2.0**-280
    st = np.zeros((5, 2, 4))
    st[:3, 0, 0] = [1, 2 * m, 2 * (2.0**-565 + m * m)]
    st[:3, 1, 0] = [1, 0.0, 2.0**-564]
    # zero variances: mean 3 vs mean 0 (t = inf), and equal means (t = NaN)
    st[:3, 0, 1] = [2, 6.0, 18.0]
    st[:3, 1, 1] = [0, 0.0, 0.0]
    st[:3, 0, 2] = [2, 6.0, 18.0]
    st[:3, 1, 2] = [2, 6.0, 18.0]
    # an ordinary point
    st[:3, 0, 3] = [2, 3.0, 7.25]
    st[:3, 1, 3] = [1, 1.0, 2.5]
    scores, pvals, lfc, pts, pts_rest = _score(st, [2, 2], 4, 0)
    assert 2.0**-564 * 2.0**-564 == 0.0 and scores[0, 0] == 4.0
    want = _p_ref(scores[0, 0], 1.0)
    assert abs(pvals[0, 0] - float(want)) <= 1e-13 * float(want) and 0.05 < pvals[0, 0] < 0.5
    assert scores[0, 1] == np.inf and pvals[0, 1] == 0.0
    assert scores[0, 2] == 0.0 and pvals[0, 2] == 1.0
    np.testing.assert_array_equal(pts[0], st[0, 0] / 2)
    np.testing.assert_array_equal(pts_rest[0], st[0, 1] / 2)
    # t-test_overestim_var: the group's n for the rest, against scipy's Welch test
    n0, n1 = 30, 400
    rng = np.random.default_rng(2)
    st = np.zeros((5, 2, 64))
    st[1] = rng.integers(-50, 200, size=(2, 64)) * 0.125
    st[2] = (st[1] ** 2 / np.array([[n0], [n1]])) + rng.integers(1, 500, size=(2, 64)) * 0.5
    for flags, nobs2 in ((0, n1), (RANK_OVERESTIM_VAR, n0)):
        scores, pvals, *_ = _score(st, [n0, n1], n0 + n1, flags)
        mg, mr = st[1, 0] / n0, st[1, 1] / n1
        vg = (st[2, 0] / n0 - mg**2) * n0 / (n0 - 1)
        vr = (st[2, 1] / n1 - mr**2) * n1 / (n1 - 1)
        want = S.ttest_ind_from_stats(mg, np.sqrt(vg), n0, mr, np.sqrt(vr), nobs2, equal_var=False)
        np.testing.assert_allclose(scores[0], want.statistic, rtol=1e-13)
        np.testing.assert_allclose(pvals[0], want.pvalue, rtol=1e-12)
    # log fold changes
    for base in (None, 2.0, 10.0):
        _, _, lfc, _, _ = _score(st, [n0, n1], n0 + n1, 0, 0.0 if base is None else float(np.log(base)))
        e = (lambda x: np.expm1(x * np.log(base))) if base is not None else np.expm1
        want = np.log2((e(st[1, 0] / n0) + 1e-9) / (e(st[1, 1] / n1) + 1e-9))
        np.testing.assert_allclose(lfc[0], want, rtol=1e-12, atol=1e-12)


# ---- 1f: the benchmark's matrix, sampled -----------------------------------------------------------------------------
def test_benchmark_shape_sampled(cuda):
    """profiles/bench_rank.py's matrix (density 0.03, 64 topics, TF-IDF) at 500 000 cells and 1500 peaks: each of its
    four configurations runs, and peak_stats on 64 sampled peaks -- the longest, and peaks on both sides of 16 384
    entries -- equals the oracle exactly, against the rest and against group "0"."""
    import muon_b200 as mu
    from muon_b200 import _device, _synth
    n, d = 500_000, 1500
    tb = _synth.make_tables(d, 0.03, 64, 0)
    A = _synth.generate_device(n, d, 0.03, tables=tb)
    X = _device.tfidf_csr(A, inplace_values=True) or A
    topics = tb.rows(0, n)[0]
    ad = mu.SimpleAnnData(shape=(n, d), obs=pd.DataFrame({"topic": pd.Categorical(
        [str(t) for t in topics], categories=[str(t) for t in range(64)])}))
    ad.X = X
    counts = torch.bincount(X.indices, minlength=d).cpu().numpy()
    cap = int(load().mub_rank_shared_capacity(4))
    assert (counts > cap).any() and ((counts > 2048) & (counts <= cap)).any()
    for kw in ({}, {"method": "wilcoxon"}, {"method": "wilcoxon", "tie_correct": True},
               {"method": "wilcoxon", "reference": "0"}):
        _rank.rank_genes_groups(ad, "topic", **kw)
        res = ad.uns["rank_genes_groups"]
        for g in res["pvals"].dtype.names:
            assert np.all((res["pvals"][g] >= 0) & (res["pvals"][g] <= 1)) and np.all(np.isfinite(res["scores"][g]))
    order = np.argsort(counts, kind="stable")
    below = order[(counts[order] > 2048) & (counts[order] <= cap)][-24:]          # the full class's longest
    above = order[counts[order] > cap][:24]                                       # the long path's shortest
    core = np.unique(np.concatenate([[order[-1]], below, above]))
    rng = np.random.default_rng(0)
    sample = np.sort(np.concatenate([core, rng.choice(np.setdiff1d(np.arange(d), core), 64 - core.size,
                                                      replace=False)]))
    Xh = X.get()
    T = sp.csr_matrix(Xh[:, sample].T)
    for reference, groups in (("rest", "all"), ("0", "all")):
        plan = _plan(topics, 64, groups, reference)
        st, share, _ = _rank.peak_stats(X, plan, sample, wilcoxon=True, tie_correct=True)
        assert 0 < share < 1
        _check(st, _oracle(T, plan, topics), plan)
