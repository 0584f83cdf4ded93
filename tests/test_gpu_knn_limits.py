"""GPU: the exact kNN kernels (csrc/knn_tc.cu, csrc/knn.cu) against float64 at the shapes and limits where they can
go wrong -- many query tiles per CTA, both operand formats and the dimensions around their switch, k at and above
the SIMT kernel's limit, crowded TF32 error bands, exact ties and the edges of the C ABI.

The tensor-core kernel is called through the C ABI (``mub_knn_l2_tc_f32``) so that the fallback inside ``knn_l2``
cannot hide a failure; ``knn_l2`` is tested on its own."""
import numpy as np
import pytest
import torch

from muon_b200 import _device
from muon_b200._lib import MuonB200Error, call, load, ptr, stream_ptr

pytestmark = pytest.mark.gpu

TC_K_MAX, SIMT_K_MAX = 512, 320


def _tc(X, k, Y=None, nq=None, nc=None, d=None, ld=None, ws_fill=None):
    """mub_knn_l2_tc_f32 on row-major buffers (``ld`` floats per row); returns (idx, dist, status word).
    ``ws_fill``: int32 value the workspace holds before the call (default: whatever the allocator returns)."""
    Y = X if Y is None else Y
    nq = X.shape[0] if nq is None else nq
    nc = Y.shape[0] if nc is None else nc
    d = X.shape[1] if d is None else d
    ld = X.shape[1] if ld is None else ld
    idx = torch.empty((nq, k), dtype=torch.int32, device=X.device)
    dist = torch.empty((nq, k), dtype=torch.float32, device=X.device)
    nbytes = int(load().mub_knn_l2_tc_workspace_bytes(nq, nc, d))
    ws = torch.empty((max(nbytes, 4) + 3) // 4, dtype=torch.int32, device=X.device)
    if ws_fill is not None:
        ws.fill_(ws_fill)
    status = torch.zeros(1, dtype=torch.int32, device=X.device)
    call("mub_knn_l2_tc_f32", ptr(X), nq, ptr(Y), nc, d, ld, k, ptr(idx), ptr(dist), ptr(ws), nbytes, ptr(status),
         stream_ptr())
    return idx, dist, int(status[0])


def _simt(X, k, Y=None, nq=None, nc=None, d=None, ld=None):
    """mub_knn_l2_f32 with an explicit row stride."""
    Y = X if Y is None else Y
    nq = X.shape[0] if nq is None else nq
    nc = Y.shape[0] if nc is None else nc
    d = X.shape[1] if d is None else d
    ld = X.shape[1] if ld is None else ld
    idx = torch.empty((nq, k), dtype=torch.int32, device=X.device)
    dist = torch.empty((nq, k), dtype=torch.float32, device=X.device)
    call("mub_knn_l2_f32", ptr(X), nq, ptr(Y), nc, d, ld, k, ptr(idx), ptr(dist), stream_ptr())
    return idx, dist


def _same(a, b):
    """Identical indices and identical distance bits."""
    return torch.equal(a[0], b[0]) and torch.equal(a[1].view(torch.int32), b[1].view(torch.int32))


def _clustered(n, d, seed, scale=3.0, n_clusters=30, normalise=True):
    """Gaussian clusters, L2-normalised rows (the WNN embeddings, as generated in profiles/bench_wnn.py)."""
    rng = np.random.default_rng(seed)
    c = rng.integers(0, n_clusters, n)
    R = rng.normal(size=(n, d)).astype(np.float32) + \
        scale * (np.eye(n_clusters, dtype=np.float32)[c] @ rng.normal(size=(n_clusters, d)).astype(np.float32))
    if normalise:
        R /= np.linalg.norm(R, axis=1, keepdims=True)
    return np.ascontiguousarray(R, dtype=np.float32)


def _sample_rows(nq, rng, n_random=480):
    """First and last rows, every row of the last partial 128-query tile, random rows."""
    tail = np.arange(nq // 128 * 128, nq)
    rows = np.concatenate([[0, nq - 1], tail, rng.choice(nq, min(n_random, nq), replace=False)])
    return np.unique(rows)


def _exact_sq(X, Y, rows, k, margin=256, block=64):
    """float64 squared distances of the (k + margin) nearest rows of Y for every X[rows], sorted by (distance,
    index): the Gram form |x|^2 + |y|^2 - 2 x.y in row blocks to shortlist, direct differences to settle."""
    Y64 = Y.astype(np.float64)
    yn = np.einsum("ij,ij->i", Y64, Y64)
    m = min(Y.shape[0], k + margin)
    out_i = np.empty((len(rows), m), dtype=np.int64)
    out_d = np.empty((len(rows), m))
    for b0 in range(0, len(rows), block):
        Q = X[rows[b0:b0 + block]].astype(np.float64)
        G = np.einsum("ij,ij->i", Q, Q)[:, None] + yn[None, :] - 2.0 * Q @ Y64.T
        sl = np.argpartition(G, m - 1, axis=1)[:, :m] if m < Y.shape[0] else np.broadcast_to(np.arange(m), G.shape)
        D2 = ((Q[:, None, :] - Y64[sl]) ** 2).sum(-1)
        o = np.lexsort((sl, D2), axis=1)
        out_i[b0:b0 + block] = np.take_along_axis(sl, o, 1)
        out_d[b0:b0 + block] = np.take_along_axis(D2, o, 1)
    return out_i, out_d


def _check_f64(X, Y, rows, idx, dist, k):
    """The kernel's rows ``rows`` against float64: same neighbour sets where the k-th and (k+1)-th distances are
    not within fp32 rounding of each other (and never a neighbour farther than the true k-th), returned distances =
    true distances of the returned indices, ascending rows, -1 / inf padding beyond the candidate count."""
    idx, dist = idx[rows], dist[rows]
    nc = Y.shape[0]
    kv = min(k, nc)
    assert np.all(idx[:, kv:] == -1) and np.all(np.isposinf(dist[:, kv:]))
    if kv == 0:
        return
    idx, dist = idx[:, :kv], dist[:, :kv]
    assert np.all(idx >= 0) and np.all(idx < nc)
    assert np.all(np.diff(dist, axis=1) >= 0)
    assert all(len(set(r)) == kv for r in idx.tolist())
    ti, td = _exact_sq(X, Y, rows, kv)
    true = np.sqrt(((X[rows][:, None, :].astype(np.float64) - Y[idx].astype(np.float64)) ** 2).sum(-1))
    np.testing.assert_allclose(dist, true, rtol=2e-6, atol=1e-30)
    kth = np.sqrt(td[:, kv - 1])
    assert np.all(true.max(axis=1) <= kth * (1 + 4e-6))           # nothing beyond the k-th nearest
    if kv < nc:
        nxt = np.sqrt(td[:, kv])
        clear = (nxt - kth) > 4e-6 * nxt
        same = np.array([set(a) == set(b) for a, b in zip(idx.tolist(), ti[:, :kv].tolist())])
        assert same[clear].all()


# ---- 1. many query tiles per CTA ----------------------------------------------------------------------------------
@pytest.mark.parametrize("d,scale", [(50, 3.0), (80, 1.0)])
def test_many_query_tiles_per_cta(cuda, d, scale):
    """n = 4 x (2 SMs) x 128 + 77 queries: every CTA of the candidate grid (2 per SM, 128 queries each) runs at
    least four query tiles, and the last tile is partial -- the per-CTA buffers and the tile counter are reused
    across tiles (the early exit of a declined call is test_declined_call_with_many_query_tiles_per_cta).  d = 50 runs the 3xTF32 operands, d = 80 the plain TF32 ones.  The d = 80 data has
    less separated clusters (scale 1) than profiles/bench_wnn.py generates: at scale 3 and d = 80 the tensor-core
    pass declines the call (status bit 2, SIMT fallback in knn_l2)."""
    sms = torch.cuda.get_device_properties(cuda).multi_processor_count
    n, k = 4 * 2 * sms * 128 + 77, 201
    R = _clustered(n, d, seed=d, scale=scale)
    X = torch.from_numpy(R).to(cuda)
    tc = _tc(X, k)
    assert tc[2] == 0, f"the tensor-core pass declined the data (status {tc[2]})"
    simt = _simt(X, k)
    assert _same(tc[:2], simt)
    rows = _sample_rows(n, np.random.default_rng(d))
    _check_f64(R, R, rows, tc[0].cpu().numpy(), tc[1].cpu().numpy(), k)
    whole = _device.knn_l2(X, k)
    chunked = _device.knn_l2(X, k, query_chunk=131072)
    assert _same(whole, chunked) and _same(whole, simt)


def test_declined_call_with_many_query_tiles_per_cta(cuda):
    """A crowded error band on every query (one tight cluster far from the origin) with four query tiles per CTA:
    the first tiles set status bit 2 and every CTA then skips its remaining tiles without writing their candidate
    lists.  The re-rank still runs on every row, so a skipped row must come out empty (-1 / inf), not built from
    whatever the workspace held -- here a count of 1 and candidate index 1 in every int32 of the workspace.  knn_l2
    returns exactly the SIMT answer."""
    sms = torch.cuda.get_device_properties(cuda).multi_processor_count
    n, d, k = 4 * 2 * sms * 128 + 77, 32, 16
    rng = np.random.default_rng(12)
    u = rng.normal(size=d)
    R = (10.0 * u / np.linalg.norm(u) + 1e-2 * rng.normal(size=(n, d))).astype(np.float32)
    X = torch.from_numpy(R).to(cuda)
    idx, dist, status = _tc(X, k, ws_fill=1)
    assert status & 2
    valid = (idx >= 0).sum(1)
    assert bool(torch.all((valid == 0) | (valid == k)))             # a row is either re-ranked in full or empty
    assert bool(torch.all(torch.isinf(dist) == (idx < 0)))
    assert int((valid == 0).sum()) > 0                                # some query tiles were skipped
    simt = _simt(X, k)
    assert _same(_device.knn_l2(X, k), simt)
    rows = _sample_rows(n, rng, n_random=64)
    _check_f64(R, R, rows, simt[0].cpu().numpy(), simt[1].cpu().numpy(), k)


# ---- 2. dimensions around the operand-format switch ----------------------------------------------------------------
@pytest.mark.parametrize("k", [1, 16, 201])
@pytest.mark.parametrize("d", [1, 3, 63, 64, 65, 79, 80, 100, 127, 128])
def test_dimension_boundaries(cuda, d, k):
    """3xTF32 for d <= 64, plain TF32 above; K padded to a multiple of 8 (Kp) on both.  nq = 1999 is not a
    multiple of 128, and every other case searches a different candidate set (nc = 2345)."""
    nq = 1999
    cross = (d + k) % 2 == 1
    nc = 2345 if cross else nq
    R = _clustered(nq + (nc if cross else 0), d, seed=1000 * d + k, scale=2.0, n_clusters=9, normalise=d > 3)
    Xh, Yh = (R[:nq], R[nq:]) if cross else (R, R)
    X, Y = torch.from_numpy(np.ascontiguousarray(Xh)).to(cuda), torch.from_numpy(np.ascontiguousarray(Yh)).to(cuda)
    tc = _tc(X, k, Y)
    assert tc[2] == 0
    simt = _simt(X, k, Y)
    assert _same(tc[:2], simt)
    rows = _sample_rows(nq, np.random.default_rng(d), n_random=256)
    _check_f64(Xh, Yh, rows, simt[0].cpu().numpy(), simt[1].cpu().numpy(), k)


# ---- 3. k at and above the SIMT kernel's limit ---------------------------------------------------------------------
def test_k_at_and_above_the_simt_limit(cuda):
    n, d = 3000, 40
    R = _clustered(n, d, seed=3)
    X = torch.from_numpy(R).to(cuda)
    rows = _sample_rows(n, np.random.default_rng(3))
    simt = _simt(X, SIMT_K_MAX)                                       # ~198 KB of shared memory per CTA
    _check_f64(R, R, rows, simt[0].cpu().numpy(), simt[1].cpu().numpy(), SIMT_K_MAX)
    tc = _tc(X, SIMT_K_MAX)
    assert tc[2] == 0 and _same(tc[:2], simt)
    for k in (SIMT_K_MAX + 1, 400, TC_K_MAX):
        tc = _tc(X, k)
        assert tc[2] == 0
        _check_f64(R, R, rows, tc[0].cpu().numpy(), tc[1].cpu().numpy(), k)
        assert _same(_device.knn_l2(X, k), tc[:2])
    with pytest.raises(MuonB200Error):
        _tc(X, TC_K_MAX + 1)
    with pytest.raises(MuonB200Error):
        _simt(X, SIMT_K_MAX + 1)
    with pytest.raises(NotImplementedError):
        _device.knn_l2(X, TC_K_MAX + 1)
    with pytest.raises(NotImplementedError):
        _device.knn_l2(X, SIMT_K_MAX + 1, algo="simt")


# ---- 4. crowded error bands ------------------------------------------------------------------------------------------
def _slack(qn, cmax, split):
    """Width of the candidate band above the k-th smallest key (knn_tc.cu: slack_rel and the per-query slack)."""
    slack_rel = 1.2e-4 if split else 4 * 2.0 ** -8
    return slack_rel * np.sqrt(qn) * cmax + 1e-5 * (qn + cmax * cmax)


@pytest.mark.parametrize("d", [32, 96])
def test_crowded_error_band_is_declined_never_wrong(cuda, d):
    """One tight cluster (spread 1e-2) at a growing distance from the origin.  The band of candidates whose TF32
    score cannot be told apart from the k-th grows with |q||c|, so the sweep runs from accepted to declined.  Every
    case must either set status bit 2 or return exactly the SIMT answer; a declined input makes knn_l2 return the
    SIMT answer, or raise for k > 320."""
    n, k = 2000, 16
    rng = np.random.default_rng(d)
    u = rng.normal(size=d)
    u /= np.linalg.norm(u)
    split = d <= 64
    accepted_wide, declined = [], []
    for off in (0.0, 0.1, 0.3, 1.0, 1.5, 3.0, 10.0, 30.0, 100.0):
        R = (off * u + 1e-2 * rng.normal(size=(n, d))).astype(np.float32)
        X = torch.from_numpy(R).to(cuda)
        tc = _tc(X, k)
        simt = _simt(X, k)
        rows = _sample_rows(n, rng, n_random=128)
        _check_f64(R, R, rows, simt[0].cpu().numpy(), simt[1].cpu().numpy(), k)
        if tc[2] & 2:
            declined.append(off)
            assert _same(_device.knn_l2(X, k), simt)
            with pytest.raises(NotImplementedError):
                _device.knn_l2(X, 400)
            continue
        assert tc[2] == 0 and _same(tc[:2], simt), f"offset {off}: accepted with a wrong answer"
        # candidates within the slack of the k-th float64 distance, per query
        R64 = R.astype(np.float64)
        nrm = np.einsum("ij,ij->i", R64, R64)
        D2 = nrm[:, None] + nrm[None, :] - 2.0 * R64 @ R64.T
        kth = np.partition(D2, k - 1, axis=1)[:, k - 1]
        band = (D2 <= (kth + _slack(nrm, np.sqrt(nrm.max()), split))[:, None]).sum(1)
        if np.percentile(band, 75) > 2 * k:
            accepted_wide.append(off)
    assert declined, "no offset was declined"
    assert accepted_wide, "no accepted offset had more than 2k candidates in its band"
    assert max(accepted_wide) < min(declined)


# ---- 5. exact ties ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k", [16, 201])
def test_exact_ties_on_a_lattice(cuda, k):
    """Integer lattice points (exact in TF32, so every score is exact and equal distances are exact ties) and
    repeated rows: ascending distance, then lower index, identical to SIMT and to a float64 stable sort."""
    rng = np.random.default_rng(k)
    L = rng.integers(-2, 3, size=(1500, 8)).astype(np.float32)
    R = np.concatenate([L, np.repeat(L[:150], 3, axis=0)])[rng.permutation(1950)]
    X = torch.from_numpy(np.ascontiguousarray(R)).to(cuda)
    tc = _tc(X, k)
    assert tc[2] == 0
    simt = _simt(X, k)
    assert _same(tc[:2], simt)
    Ri = R.astype(np.int64)
    n2 = (Ri * Ri).sum(1)
    D2 = n2[:, None] + n2[None, :] - 2 * Ri @ Ri.T                    # exact in integers
    order = np.argsort(D2, axis=1, kind="stable")[:, :k]
    np.testing.assert_array_equal(tc[0].cpu().numpy(), order)
    np.testing.assert_array_equal(tc[1].cpu().numpy(), np.sqrt(np.take_along_axis(D2, order, 1).astype(np.float32)))


# ---- 6. edges of the C ABI ----------------------------------------------------------------------------------------
def test_row_stride_wider_than_d(cuda):
    """ld > d: the rows are views into a wider buffer whose extra columns hold NaN, so any read past d shows."""
    nq, nc, k = 700, 900, 24
    for d in (20, 80):
        R = _clustered(nq + nc, d, seed=d, n_clusters=9)
        for extra in (1, 13):
            W = torch.full((nq + nc, d + extra), float("nan"), device=cuda)
            W[:, :d] = torch.from_numpy(R).to(cuda)
            X, Y = W[:nq], W[nq:]
            dense = torch.from_numpy(R[:nq].copy()).to(cuda), torch.from_numpy(R[nq:].copy()).to(cuda)
            ref = _simt(dense[0], k, dense[1])
            tc = _tc(X, k, Y, d=d, ld=d + extra)
            assert tc[2] == 0 and _same(tc[:2], ref)
            assert _same(_simt(X, k, Y, d=d, ld=d + extra), ref)
        rows = np.arange(nq)
        _check_f64(R[:nq], R[nq:], rows, ref[0].cpu().numpy(), ref[1].cpu().numpy(), k)


def test_no_candidates_no_queries_and_a_single_partial_tile(cuda):
    d, k = 16, 8
    R = _clustered(300, d, seed=6, n_clusters=5)
    X = torch.from_numpy(R).to(cuda)
    # nc = 0: every slot is padding
    for run in (_tc, _simt):
        out = run(X, k, X, nc=0)
        assert torch.all(out[0] == -1) and torch.all(torch.isinf(out[1])) and torch.all(out[1] > 0)
    # nq = 0: nothing is written
    idx = torch.full((4, k), 7, dtype=torch.int32, device=cuda)
    dist = torch.full((4, k), 3.0, device=cuda)
    nbytes = int(load().mub_knn_l2_tc_workspace_bytes(0, 300, d))
    ws = torch.empty(max(nbytes, 4), dtype=torch.uint8, device=cuda)
    status = torch.zeros(1, dtype=torch.int32, device=cuda)
    call("mub_knn_l2_tc_f32", ptr(X), 0, ptr(X), 300, d, d, k, ptr(idx), ptr(dist), ptr(ws), nbytes, ptr(status),
         stream_ptr())
    call("mub_knn_l2_f32", ptr(X), 0, ptr(X), 300, d, d, k, ptr(idx), ptr(dist), stream_ptr())
    torch.cuda.synchronize()
    assert torch.all(idx == 7) and torch.all(dist == 3.0) and int(status[0]) == 0
    # nq < 128: one partial query tile, against the whole set
    for nq in (1, 37, 127):
        tc = _tc(X[:nq], k, X)
        assert tc[2] == 0 and _same(tc[:2], _simt(X[:nq], k, X))
        _check_f64(R[:nq], R, np.arange(nq), tc[0].cpu().numpy(), tc[1].cpu().numpy(), k)
