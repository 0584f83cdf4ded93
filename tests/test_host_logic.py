"""CPU: host-side logic above the C ABI -- containers, argument checking, the block
Golub-Kahan driver (with a scipy operator injected by the test; the product wires CUDA)."""
import numpy as np
import pytest
import scipy.sparse as sp
import torch

import muon_b200 as mu
from conftest import golden_csr, load_golden
from muon_b200._containers import SimpleAnnData, SimpleMuData, view_to_actual
from muon_b200._lsi import truncated_svd
from muon_b200._synth import generate_host, make_tables
from oracle.lsi_ref import compare_lsi, lsi_ref
from oracle.tfidf_ref import tfidf_ref


class ScipyOperator:
    """Test-only stand-in for CsrOperator (same protocol: av, aty, gram)."""

    def __init__(self, A):
        self.A = sp.csr_matrix(A).astype(np.float32)
        self.At = self.A.T.tocsr()
        self.n_local, self.d = self.A.shape
        self.n_total = self.n_local
        self.device = torch.device("cpu")

    def av(self, V):
        return torch.from_numpy(self.A @ V.numpy())

    def aty(self, Y):
        return torch.from_numpy(self.At @ Y.numpy())

    def gram(self, Y, l):
        y = Y[:, :l].double()
        return y.T @ y


class SamplingOperator(ScipyOperator):
    """ScipyOperator with the optional residual_sample hook (here on every 4th peak)."""

    def __init__(self, A):
        super().__init__(A)
        self.samples = 0

    def residual_sample(self, Uk, Vk, sig):
        self.samples += 1
        k = Vk.shape[1]
        idx = np.arange(0, self.d, 4)
        W = (self.At[idx] @ Uk.numpy())[:, :k]
        R = W.astype(np.float64) - Vk.numpy()[idx].astype(np.float64) * sig.numpy()[None, :k]
        return torch.from_numpy(np.sqrt((R * R).sum(0) * (self.d / idx.size)) / sig.numpy()[:k])


def test_containers_view_copy_slots():
    x = np.arange(20, dtype=float).reshape(4, 5)
    ad = SimpleAnnData(x)
    v = ad[:, :]
    assert v.is_view
    view_to_actual(v)
    assert not v.is_view and v.X is not ad.X
    c = ad.copy()
    c.X[0, 0] = -1
    assert ad.X[0, 0] == 0
    with pytest.raises(ValueError):
        ad.X = np.zeros((3, 3))
    md = SimpleMuData({"atac": ad, "rna": SimpleAnnData(np.ones((4, 3)))})
    assert md.n_obs == 4 and md.n_vars == 8 and "atac" in md.mod


def test_tfidf_argument_errors_match_reference():
    # muon/_atac/preproc.py:62-79 -- raised before any device work
    ad = SimpleAnnData(np.ones((3, 3)))
    with pytest.raises(TypeError):
        mu.atac.pp.tfidf(np.ones((3, 3)))
    with pytest.raises(TypeError):
        mu.atac.pp.tfidf(SimpleMuData({"rna": ad}))
    with pytest.raises(AttributeError):
        mu.atac.pp.tfidf(ad, log_tfidf=True)
    with pytest.raises(ValueError):
        mu.atac.pp.tfidf(ad, copy=True, inplace=False)
    with pytest.raises(ValueError):
        mu.atac.pp.tfidf(ad, to_layer="x", inplace=False)
    with pytest.raises(TypeError):
        mu.atac.tl.lsi(np.ones((3, 3)))


def test_no_cpu_fallback():
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from muon_b200._lib import MuonB200Error
    ad = SimpleAnnData(sp.random(20, 10, 0.3, format="csr", random_state=0))
    with pytest.raises(MuonB200Error):
        mu.atac.pp.tfidf(ad)
    with pytest.raises(MuonB200Error):
        mu.atac.tl.lsi(ad, n_comps=3)


@pytest.mark.parametrize("k,P", [(8, 32), (20, 32), (30, 64)])
def test_block_lanczos_ritz_triplets_from_the_left_blocks_match_svds(k, P):
    """U_k read off the stored left Lanczos blocks, s and V_k meet the float64 svds parity bar, and U_k is
    orthonormal."""
    X = tfidf_ref(generate_host(1500, 1200, 0.05, n_topics=12, seed=3)).astype(np.float32)
    ref = lsi_ref(X, k + 1, dtype=np.float64)
    s_next = ref["svalues"][k]
    ref = {"svalues": ref["svalues"][:k], "U": ref["U"][:, :k], "LSI": ref["LSI"][:, :k]}
    U, s, V, info = truncated_svd(ScipyOperator(X), k, P, tol=1e-5)
    assert info.converged
    out = compare_lsi({"svalues": s.numpy(), "U": U.numpy(), "LSI": V.numpy()}, ref, rtol=1e-4, s_next=s_next)
    assert out["sigma_rel"] < 1e-5
    assert np.abs(U.numpy().T.astype(np.float64) @ U.numpy() - np.eye(k)).max() < 1e-5


def test_block_lanczos_small_dims_and_restart():
    # d smaller than the kernel width, and a basis cap that forces a restart
    X = sp.random(300, 20, 0.4, format="csr", random_state=1, dtype=np.float32)
    ref = lsi_ref(X, 5, dtype=np.float64)
    U, s, V, info = truncated_svd(ScipyOperator(X), 5, 32)
    np.testing.assert_allclose(s.numpy(), ref["svalues"], rtol=1e-5)
    X = tfidf_ref(generate_host(800, 900, 0.05, n_topics=8, seed=4)).astype(np.float32)
    ref = lsi_ref(X, 6, dtype=np.float64)
    U, s, V, info = truncated_svd(ScipyOperator(X), 6, 32, max_basis=96, max_restarts=8)
    assert info.restarts >= 1
    np.testing.assert_allclose(s.numpy(), ref["svalues"], rtol=1e-4)


def test_oracle_lsi_matches_unmodified_reference():
    z = load_golden("lsi_synth.npz")
    X = golden_csr(z, "x")
    r = lsi_ref(X, 8)
    np.testing.assert_allclose(r["stdev"], z["stdev"], rtol=1e-10)
    got = {"svalues": r["stdev"], "U": r["U"], "LSI": r["LSI"]}
    ref = {"svalues": z["stdev"], "U": z["U"], "LSI": z["LSI"]}
    compare_lsi(got, ref, rtol=1e-8)
    emb = r["X_lsi"] * np.sign((r["X_lsi"] * z["X_lsi"]).sum(0))
    np.testing.assert_allclose(emb, z["X_lsi"], rtol=0, atol=1e-7)


def test_synth_generator_is_shard_consistent():
    tb = make_tables(700, 0.05, n_topics=5, seed=9)
    full = generate_host(120, 700, 0.05, tables=tb)
    a = generate_host(50, 700, 0.05, tables=tb, row0=0)
    b = generate_host(70, 700, 0.05, tables=tb, row0=50)
    stacked = sp.vstack([a, b]).tocsr()
    np.testing.assert_array_equal(full.indptr, stacked.indptr)
    np.testing.assert_array_equal(full.indices, stacked.indices)
    np.testing.assert_array_equal(full.data, stacked.data)
    assert abs(full.nnz / (120 * 700) - 0.05) < 0.01
    assert set(np.unique(full.data)) <= {1.0, 2.0, 3.0, 4.0, 5.0}


def test_k_beyond_separated_spectrum_is_reported_not_hidden():
    """k larger than the number of planted topics: the trailing wanted components sit in the noise bulk
    (relative gaps ~1e-3), block Lanczos crawls, and the driver must say so (converged=False) instead of
    silently returning; the separated leading components are still right."""
    X = tfidf_ref(generate_host(1200, 1000, 0.05, n_topics=6, seed=21)).astype(np.float32)
    k = 24
    ref = lsi_ref(X, k, dtype=np.float64)
    U, s, V, info = truncated_svd(ScipyOperator(X), k, 32, tol=1e-7, max_basis=192, max_restarts=1)
    assert not info.converged and max(info.residuals) > 1e-7
    np.testing.assert_allclose(s.numpy()[:6], ref["svalues"][:6], rtol=1e-5)
    lead = np.abs((V.numpy()[:, :6] * ref["LSI"][:, :6]).sum(0))
    assert np.all(1 - lead < 1e-6)


def test_resident_copy_fingerprint_sees_any_single_value_edit():
    """lsi() reuses the device copy left by tfidf() only if every host element still matches what crossed the bus:
    the staging engine's fingerprint must change with any single edit, at any length (tail handling)."""
    from muon_b200 import _device as d
    pool = d.host_pool()
    for n in (1, 7, 8, 9, 1_000_003):
        a = np.random.default_rng(n).standard_normal(n).astype(np.float32)
        h = pool.fingerprint(a)
        b = a.copy()
        b[n // 3] = np.nextafter(b[n // 3], np.float32(9))
        assert pool.fingerprint(b) != h and pool.fingerprint(a.copy()) == h
    assert pool.fingerprint(np.zeros(0, dtype=np.float32)) == 0


def test_bench_onchip_roofline_arithmetic():
    import importlib.util, os
    spec = importlib.util.spec_from_file_location("bench", os.path.join(os.path.dirname(__file__), "..", "bench.py"))
    bench = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bench)
    r = bench.onchip_roofline(nnz=6_000_000_000, P=64, ms_per_pass=88.0, sm_mhz=1980.0)
    assert abs(r["peak"] - 132 * 128 * 1.98e9 / 1e12) < 1e-9 and r["bytes_per_nnz"] == 264.0
    assert abs(r["achieved"] - 6e9 * 264 / 0.088 / 1e12) < 1e-9 and 0.45 < r["frac"] < 0.55
    assert bench.onchip_roofline(1, 64, float("nan"), 1900.0) is None and bench.onchip_roofline(1, 64, 1.0, None) is None


def test_neighbors_argument_errors_and_no_cpu_fallback():
    """muon/_core/preproc.py:264-398 checks, raised before any device work; without a GPU the call must fail
    loudly instead of computing anything on the host."""
    with pytest.raises(TypeError):
        mu.pp.neighbors(np.ones((3, 3)))
    ads = {}
    for name in ("a", "b"):
        ad = SimpleAnnData(np.zeros((6, 2)))
        ad.obsm["X_e"] = np.random.default_rng(0).normal(size=(6, 3))
        ad.obsp["distances"] = sp.csr_matrix(np.ones((6, 6)) - np.eye(6))
        ad.uns["neighbors"] = {"params": {"n_neighbors": 3, "use_rep": "X_e"}, "distances_key": "distances"}
        ads[name] = ad
    md = SimpleMuData(ads)
    with pytest.raises(NotImplementedError):
        mu.pp.neighbors(md, metric="cosine")
    del md.mod["b"].uns["neighbors"]
    with pytest.raises(ValueError):
        mu.pp.neighbors(md)
    if not torch.cuda.is_available():
        from muon_b200._lib import MuonB200Error
        with pytest.raises(MuonB200Error):
            mu.pp.neighbors(SimpleMuData({k: v for k, v in ads.items() if k == "a"}))
        with pytest.raises(MuonB200Error):
            mu.tl.mofa(SimpleMuData({"y": SimpleAnnData(np.random.default_rng(1).normal(size=(20, 8)))}), n_factors=2)


class HalfOperandOperator(ScipyOperator):
    """ScipyOperator that also offers the product's low-precision mode: the dense operand of a product is rounded
    to IEEE half after the same power-of-two scaling the CUDA path uses (muon_b200._device.HALF_SCALE).  Like
    CsrOperator it has gram_local, so the driver's d-space QR is CholeskyQR2."""
    lowp = True

    def __init__(self, A):
        super().__init__(A)
        self.lowp_calls = 0
        self.gram_local_calls = 0

    def gram_local(self, Y, l):
        self.gram_local_calls += 1
        return self.gram(Y, l)

    @staticmethod
    def _round(M):
        return (M.numpy() * np.float32(32768.0)).astype(np.float16).astype(np.float32) / np.float32(32768.0)

    def av(self, V, lowp=False):
        self.lowp_calls += int(lowp)
        return torch.from_numpy(self.A @ (self._round(V) if lowp else V.numpy()))

    def aty(self, Y, lowp=False):
        self.lowp_calls += int(lowp)
        return torch.from_numpy(self.At @ (self._round(Y) if lowp else Y.numpy()))


@pytest.mark.parametrize("k,P", [(20, 32), (30, 64)])
def test_block_lanczos_half_precision_phase(k, P):
    """Two-phase schedule: half-precision operands until 1e-3, then fp32 from the Ritz vectors.  The result must
    meet the same parity bar as the all-fp32 iteration, with most passes done in the cheap mode."""
    X = tfidf_ref(generate_host(1500, 1200, 0.05, n_topics=12, seed=3)).astype(np.float32)
    ref = lsi_ref(X, k + 1, dtype=np.float64)
    s_next = ref["svalues"][k]
    ref = {"svalues": ref["svalues"][:k], "U": ref["U"][:, :k], "LSI": ref["LSI"][:, :k]}
    op = HalfOperandOperator(X)
    U, s, V, info = truncated_svd(op, k, P, tol=1e-5)
    assert info.converged and info.lowp_passes == op.lowp_calls > 0 and op.gram_local_calls > 0
    assert info.lowp_passes >= info.passes // 2, (info.lowp_passes, info.passes)
    out = compare_lsi({"svalues": s.numpy(), "U": U.numpy(), "LSI": V.numpy()}, ref, rtol=1e-4, s_next=s_next)
    assert out["sigma_rel"] < 1e-5
    # an operator without the low-precision mode runs fp32 only
    U2, s2, V2, info2 = truncated_svd(ScipyOperator(X), k, P, tol=1e-5)
    assert info2.lowp_passes == 0


def test_host_fingerprint_pool_only():
    """The staging engine's fingerprint on the host (thread pool only, no CUDA): independent of the thread count,
    position dependent, and equal for an int64 array and its int32 narrowing."""
    from muon_b200 import _device
    rng = np.random.default_rng(0)
    a = rng.integers(0, 2**31 - 1, 3_000_001, dtype=np.int64)
    h = [_device.Stager(pool_only=True, threads=t).fingerprint(a) for t in (1, 3, 8)]
    assert h[0] == h[1] == h[2] == _device.Stager(pool_only=True, threads=2).fingerprint(a.astype(np.int32))
    # the definition: sum_i u64(e_i ^ a_i) * u64(b_i) mod 2^64, a_i = u32(i*K1 + C1), b_i = u32(i*K2 + C2) | 1  (i < 2^32)
    K1, K2, C1, C2, M32, M = 0x9E3779B1, 0x85EBCA6B, 0x7F4A7C15, 0x165667B1, (1 << 32) - 1, (1 << 64) - 1
    small = [5, 0, 2**31 - 2, 77]
    want = sum((e ^ ((i * K1 + C1) & M32)) * (((i * K2 + C2) & M32) | 1) for i, e in enumerate(small)) & M
    assert _device.Stager(pool_only=True, threads=2).fingerprint(np.array(small, dtype=np.int32)) == want
    b = a.copy()
    b[[1, 2_999_999]] = b[[2_999_999, 1]]
    assert _device.host_pool().fingerprint(b) != h[0]
    f = rng.standard_normal(1000).astype(np.float32)
    assert _device.host_pool().fingerprint(f) == _device.host_pool().fingerprint(f.view(np.uint32))


def test_reference_arm_does_not_load_the_cuda_library():
    import subprocess
    import sys
    from conftest import ROOT
    code = ("import sys; sys.argv=['bench.py','--impl','reference','--sample-cells','300','--peaks','1500','--k','5',"
            "'--steps','1','--warmup','1']; import runpy; runpy.run_path('bench.py', run_name='__main__');"
            "assert 'libmuon_b200' not in open('/proc/self/maps').read(), 'reference arm loaded the CUDA library'")
    out = subprocess.run([sys.executable, "-c", code], cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stderr[-2000:]
    assert '"impl": "reference"' in out.stdout


def test_sampled_residual_check_replaces_only_the_confirming_pass():
    """When the history predicts convergence the driver estimates the residual on a sample of the peaks and skips the
    pass that would only confirm it; the result meets the same parity bar, an operator without the hook is unaffected,
    and a failed estimate falls through to the full pass."""
    k, P = 20, 32
    X = tfidf_ref(generate_host(1500, 1200, 0.05, n_topics=12, seed=3)).astype(np.float32)
    ref = lsi_ref(X, k + 1, dtype=np.float64)
    s_next = ref["svalues"][k]
    ref = {"svalues": ref["svalues"][:k], "U": ref["U"][:, :k], "LSI": ref["LSI"][:, :k]}
    U0, s0, V0, info0 = truncated_svd(ScipyOperator(X), k, P, tol=1e-5)
    op = SamplingOperator(X)
    U, s, V, info = truncated_svd(op, k, P, tol=1e-5)
    assert info0.sampled_checks == 0 and op.samples == info.sampled_checks >= 1
    if info.sampled_stop:
        assert info.passes == info0.passes - 1
    out = compare_lsi({"svalues": s.numpy(), "U": U.numpy(), "LSI": V.numpy()}, ref, rtol=1e-4, s_next=s_next)
    assert out["sigma_rel"] < 1e-5
    assert np.abs(U.numpy().T.astype(np.float64) @ U.numpy() - np.eye(k)).max() < 1e-5

    class Pessimist(SamplingOperator):
        def residual_sample(self, Uk, Vk, sig):
            return super().residual_sample(Uk, Vk, sig) * 1e3          # never accepted

    op2 = Pessimist(X)
    U2, s2, V2, info2 = truncated_svd(op2, k, P, tol=1e-5)
    assert not info2.sampled_stop and info2.passes == info0.passes and info2.converged
    np.testing.assert_allclose(s2.numpy(), s0.numpy(), rtol=1e-6)


def test_nnz_balanced_row_blocks():
    """Cell shards for multi-GPU runs are cut by stored entries, not by rows (SURVEY 8e): contiguous, covering, and
    within one row's worth of the ideal share even for very skewed depths."""
    from muon_b200._dist import balanced_row_range
    rng = np.random.default_rng(0)
    lens = np.concatenate([rng.integers(1, 20, 5000), rng.integers(2000, 9000, 300), rng.integers(1, 20, 3000)])
    indptr = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    for world in (1, 2, 3, 8):
        blocks = [balanced_row_range(indptr, world, r) for r in range(world)]
        assert blocks[0][0] == 0 and blocks[-1][1] == len(lens)
        assert all(a[1] == b[0] for a, b in zip(blocks, blocks[1:]))
        share = indptr[-1] / world
        for r0, r1 in blocks:
            assert abs((indptr[r1] - indptr[r0]) - share) <= lens.max() + 1
    assert balanced_row_range(torch.from_numpy(indptr), 2, 1) == balanced_row_range(indptr, 2, 1)


def test_row_chunk_and_upload_block_boundaries():
    """Host-side geometry the tiled kernels rely on: the 16 row chunks are aligned to the tiled kernels' block height
    (a CTA never straddles a chunk), nest into 1/2/4/8/16 panels, and the upload blocks of the host path are cut on
    the same alignment while covering every row exactly once."""
    from muon_b200 import _device
    R = _device.tile_rows()
    assert R == 512
    for n in (1, 300, 512, 5000, 20_000, 1_000_000, 1_234_567):
        cb = _device.chunk_bounds(n)
        assert len(cb) == _device.N_CHUNKS + 1 and cb[0] == 0 and cb[-1] == n
        assert all(a <= b for a, b in zip(cb, cb[1:])) and all(b % R == 0 or b == n for b in cb)
        for n_panels in (1, 2, 4, 8, 16):
            per = _device.N_CHUNKS // n_panels
            pb = [cb[i * per] for i in range(n_panels)] + [n]
            assert pb[0] == 0 and pb[-1] == n and all(a <= b for a, b in zip(pb, pb[1:]))
    rng = np.random.default_rng(0)
    lens = rng.integers(0, 4000, 7000)
    indptr = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    blocks = _device._row_blocks(indptr, 1_000_000, R)
    assert blocks[0][0] == 0 and blocks[-1][1] == 7000
    for (r0, r1, k0, k1), nxt in zip(blocks, blocks[1:] + [None]):
        assert r0 % R == 0 and r1 > r0 and k0 == indptr[r0] and k1 == indptr[r1]
        if nxt is not None:
            assert nxt[0] == r1
    assert _device._row_blocks(indptr[:1], 10, R) == []
    assert _device.sample_row_blocks(200_000) and sum(b - a for a, b in _device.sample_row_blocks(200_000)) == 200_000 // 16
