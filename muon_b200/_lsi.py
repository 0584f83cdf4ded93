"""Truncated SVD driver for LSI: block Golub-Kahan-Lanczos with Rayleigh-Ritz.

The reference computes ``svds(adata.X, k)`` (muon/_atac/tools.py:53): ARPACK ``eigsh`` on the
implicit X^T X, one vector at a time -- 300-900 single-vector passes over the matrix for
k=50 (SURVEY section 6).  On an H100 every pass streams the whole CSR from HBM, so the design
goal is *few, wide* passes: a block of ``b`` vectors (b = padded kernel width, 64 for k=50)
per pass and a Krylov method that converges in a handful of block steps.

Algorithm (host side, all heavy work in the three operator callbacks):

  V_1 = orth(randn(d, b));  U_1 R_1 = qr(A V_1)
  repeat   W = A^T U_j - V_j R_j^T                     (SpMM on A^T; allreduce over cell shards)
           W -= V_all (V_all^T W)   (x2)               (full reorthogonalisation, d-space, replicated)
           V_{j+1} S_j = qr(W)
           Y = A V_{j+1} - U_j S_j^T                   (SpMM on A; local to the cell shard)
           U_{j+1} R_{j+1} = cholqr2(Y)                (Gram kernel + b x b allreduce)
           B = blockbidiag(R, S^T);  svd(B) in fp64 -> Ritz values, residuals ||S_j x_last||
  until the first k residuals are below tol * sigma_i (or stagnate at the fp32 floor)
  V_k = V_all Z[:, :k];  Y = A V_k;  G = Y^T Y (allreduce);  eigh(G) -> sigma, U = Y Z / sigma

The last line is the same Rayleigh-Ritz polish scipy applies after ARPACK
(``eigvec -> Av -> svd(Av)``, scipy _svds.py:508-533).  Working on A (not A^T A) keeps the
attainable accuracy at eps*sigma_1/sigma_i instead of eps*(sigma_1/sigma_i)^2.

The driver is backend-agnostic: ``op`` supplies ``av``, ``aty``, ``gram``.  The product
wires the CUDA kernels (``CsrOperator``); CPU tests of this host logic inject a scipy
operator of their own.
"""
from __future__ import annotations

import os
from dataclasses import dataclass, field
from typing import Optional

import torch

from . import _dist
from ._lib import phase


@dataclass
class SvdInfo:
    passes: int = 0              # sparse passes over A or A^T
    lowp_passes: int = 0         # of which with the dense operand rounded to IEEE half
    replica_repairs: int = 0     # multi-GPU: times the replicated d-space block had to be re-broadcast (expected 0)
    sampled_checks: int = 0      # residual estimates on 1/16 of the peaks (each costs 1/16 of a pass)
    sampled_stop: bool = False   # convergence was accepted on such an estimate (<= tol/3) instead of a full pass
    iterations: int = 0
    restarts: int = 0
    basis: int = 0
    block: int = 0
    residuals: list = field(default_factory=list)   # relative residual of the k wanted triplets
    converged: bool = False      # all k residuals <= tol (or the Krylov space is the whole space)
    stalled: bool = False        # stopped because the residuals stopped improving (fp32 floor or clustered spectrum)
    history: list = field(default_factory=list)     # max relative residual per iteration


class CsrOperator:
    """A (cell shard) and A^T as CUDA SpMM + Gram kernels."""

    def __init__(self, A, pad: int = 64):
        from . import _device
        self._dev = _device
        self.A = A
        with phase("lsi.transpose"):
            self.At = A.transpose_panels(pad, side_stream=os.environ.get("MUON_B200_OVERLAP", "0") == "1")
        self.n_local, self.d = A.shape
        self.n_total = A.n_total
        self.device = A.data.device
        self.passes = 0

    lowp = True      # av / aty accept lowp=True: dense operand rounded to IEEE half (csrc/spmm.cu, spmm_row_h)

    def av(self, V, lowp: bool = False):
        self.passes += 1
        with phase("lsi.spmm_av"):
            if lowp:
                return self._dev.spmm_h16(self.A, self._dev.to_half_scaled(V), dynamic=False)
            return self._dev.spmm(self.A, V, dynamic=False)

    def aty(self, Y, lowp: bool = False):
        """A^T Y summed over the cell shards.  Multi-GPU: with $MUON_B200_AR_CHUNKS > 1 the product is computed in
        blocks of peaks and the allreduce of block c runs (NCCL stream) under the SpMM of block c+1."""
        self.passes += 1
        with phase("lsi.spmm_aty"):
            if not _dist.is_distributed():
                return self.At.spmm(Y, dynamic=True, half=lowp)
            works = []
            W = self.At.spmm(Y, dynamic=True, half=lowp, row_chunks=self.AR_CHUNKS,
                             on_chunk=lambda blk: works.append(_dist.all_reduce_sum_async(blk)))
            for w in works:
                w.wait()
            return W

    # several blocks overlap the allreduce with the product but split the SpMM into smaller, less efficient
    # launches, and the allreduce of a d x P block is short, so the default is one block (the overlapped path stays available and tested)
    AR_CHUNKS = int(os.environ.get("MUON_B200_AR_CHUNKS", "1"))

    def residual_sample(self, Uk, Vk, sig):
        """Estimate of the relative residuals ||A^T u_i - sigma_i v_i|| / sigma_i of k triplets from 1/16 of the
        peaks (4 evenly spaced contiguous blocks of rows of A^T; peak indices carry no structure): ||r||^2 ~ (d/|S|) * sum_{j in S} r_j^2.  Costs 1/16
        of a pass; the driver uses it to skip the pass that would only confirm convergence."""
        blocks = self._dev.sample_row_blocks(self.d)
        with phase("lsi.residual_sample"):
            W = self.At.spmm_rowblocks(Uk.contiguous(), blocks)          # Uk: n_local x P (padded by the driver)
            W = _dist.all_reduce_sum_(W)
            idx = torch.cat([torch.arange(j0, j1, device=self.device) for j0, j1 in blocks])
            k = Vk.shape[1]
            R = W[:, :k].to(torch.float64) - Vk[idx].to(torch.float64) * sig[None, :k]
            return torch.sqrt((R * R).sum(0) * (self.d / idx.numel())) / sig[:k].clamp_min(1e-300)

    def gram(self, Y, l):
        return self._dev.gram(Y, l, reduce=True)

    def gram_local(self, Y, l):          # replicated (d-space) operand: no allreduce
        return self._dev.gram(Y, l, reduce=False)


def _pad(M: torch.Tensor, P: int) -> torch.Tensor:
    if M.shape[1] == P and M.is_contiguous():
        return M
    out = torch.zeros((M.shape[0], P), dtype=M.dtype, device=M.device)
    out[:, :M.shape[1]] = M
    return out


def _chol_upper(G: torch.Tensor) -> torch.Tensor:
    """Upper Cholesky factor of a (nearly) SPD fp64 Gram; shifted retry if rounding broke SPD."""
    G = 0.5 * (G + G.T)
    L, info = torch.linalg.cholesky_ex(G)
    shift = 0.0
    scale = float(torch.diagonal(G).abs().max())
    while int(info) != 0:
        shift = max(shift * 10.0, 1e-10 * scale)
        L, info = torch.linalg.cholesky_ex(G + shift * torch.eye(G.shape[0], dtype=G.dtype, device=G.device))
        if shift > 1e-2 * scale:
            raise RuntimeError("CholeskyQR: Gram matrix is numerically singular")
    return L.T


def _cholqr2(op, Y: torch.Tensor, l: int):
    """Y[n x P] (first l columns meaningful) -> Q (same layout, orthonormal over all shards), R[l x l] fp64."""
    R_tot = None
    for _ in range(2):
      with phase("lsi.cholqr"):
        G = op.gram(Y, l)
        R = _chol_upper(G)
        Rinv = torch.linalg.solve_triangular(R, torch.eye(l, dtype=R.dtype, device=R.device), upper=True)
        M = torch.zeros((Y.shape[1], Y.shape[1]), dtype=torch.float32, device=Y.device)
        M[:l, :l] = Rinv.to(torch.float32)
        Y = Y @ M
        R_tot = R if R_tot is None else R @ R_tot
    return Y, R_tot


def _qr_dspace(op, W: torch.Tensor, P: int):
    """Thin QR of a replicated d x b block.  CholeskyQR2 on the Gram kernel when the operator has
    one and the block is well conditioned (0.3 ms instead of ~5 ms of Householder panels for
    200k x 64); Householder (cuSOLVER geqrf) otherwise."""
    gl = getattr(op, "gram_local", None)
    l = W.shape[1]
    if gl is not None and l <= P and W.shape[0] >= 4 * l:
        Wp = _pad(W, P)
        R_tot = None
        ok = True
        for _ in range(2):
            G = gl(Wp, l)
            G = 0.5 * (G + G.T)
            L, info = torch.linalg.cholesky_ex(G)
            dg = torch.diagonal(L)
            if int(info) != 0 or float(dg.min()) < 1e-4 * float(dg.max()):   # cond(W) > ~1e4: not safe in fp32
                ok = False
                break
            R = L.T
            Rinv = torch.linalg.solve_triangular(R, torch.eye(l, dtype=R.dtype, device=R.device), upper=True)
            M = torch.zeros((P, P), dtype=torch.float32, device=W.device)
            M[:l, :l] = Rinv.to(torch.float32)
            Wp = Wp @ M
            R_tot = R if R_tot is None else R @ R_tot
        if ok:
            return Wp[:, :l], R_tot.to(torch.float32)
    return torch.linalg.qr(W)


def _orth_against(W: torch.Tensor, Q: torch.Tensor, passes: int = 2):
    """Classical Gram-Schmidt (x passes) of W against the orthonormal columns of Q; returns the
    accumulated coefficients Q^T W in fp64."""
    H = torch.zeros((Q.shape[1], W.shape[1]), dtype=torch.float64, device=W.device)
    for _ in range(passes):
        h = Q.T @ W
        W -= Q @ h
        H += h.to(torch.float64)
    return W, H


def truncated_svd(op, k: int, pad_to: int, tol: float = 1e-5, max_basis: Optional[int] = None,
                  max_restarts: int = 4, seed: int = 0, verbose: bool = False, polish: Optional[bool] = None,
                  lowp_tol: Optional[float] = None, sample_check: Optional[bool] = None):
    """Top-k singular triplets of the (cell-sharded) matrix behind ``op``.

    Returns (U [n_local x k] fp32, s [k] fp64, V [d x k] fp32, SvdInfo).  ``pad_to`` is the padded
    dense width the kernels run at (32/64/128); the Krylov block size is min(pad_to, d).

    ``polish`` (default: $MUON_B200_LSI_POLISH, "0"): finish with scipy's Rayleigh-Ritz tail (one more pass over A).
    ``False`` returns the Ritz triplets of the Krylov spaces themselves -- U_k from the stored left blocks -- and
    saves that pass; both meet the same parity bar on the CPU driver tests and on the GPU suite (sigma 1e-7, vectors
    < 1e-5 against float64 svds; tests/test_gpu_round2.py), so the cheaper one is the default since round 2.

    ``lowp_tol`` (default: $MUON_B200_LSI_LOWP_TOL, "1e-3"; "0" = off): if > ``tol`` and the operator supports it
    (``op.lowp``), the iteration first runs with the dense operand of every product rounded to IEEE half -- half the
    bytes through the gather path that bounds the SpMM kernel -- until the wanted triplets reach ``lowp_tol``
    (rounding to half caps the attainable residual near 2e-4, so 1e-3 is the useful setting), then restarts in
    fp32 from the Ritz vectors: one fp32 block step takes residuals from ~3e-4 to below 1e-5.  The result is the
    fp32 iteration's own (same stopping rule, same Rayleigh-Ritz tail); only the path to the final subspace is
    cheaper.  ``SvdInfo.lowp_passes`` counts the half-precision passes.

    ``sample_check`` (default: $MUON_B200_LSI_SAMPLE_CHECK, "1"): when the residual history predicts that the next
    pass over A^T would only confirm convergence, estimate the residuals on 1/16 of the peaks first
    (``op.residual_sample``) and stop if the estimate is <= tol/2; the full pass is skipped only then.
    """
    if polish is None:
        polish = os.environ.get("MUON_B200_LSI_POLISH", "0") != "0"
    if lowp_tol is None:
        lowp_tol = float(os.environ.get("MUON_B200_LSI_LOWP_TOL", "1e-3") or 0.0)
    lowp = bool(getattr(op, "lowp", False)) and lowp_tol > tol
    if sample_check is None:
        sample_check = os.environ.get("MUON_B200_LSI_SAMPLE_CHECK", "1") != "0"
    d, dev, P = op.d, op.device, pad_to
    k = int(k)
    b = min(P, d, getattr(op, "n_total", d))
    assert 1 <= k <= b, (k, b)
    m_cap = min(d, max_basis if max_basis is not None else 16 * P)
    m_cap = max(m_cap, min(d, 2 * b))
    info = SvdInfo(block=b)
    f64 = torch.float64

    with phase("lsi.init"):
        g = torch.Generator(device=dev).manual_seed(int(seed))   # same stream on every rank (same device type)
        V0 = torch.randn((d, b), generator=g, dtype=torch.float32, device=dev)
        V0, _ = _qr_dspace(op, V0, P)

    def _av(V):
        return op.av(V, lowp=True) if lowp else op.av(V)

    def _aty(Y):
        return op.aty(Y, lowp=True) if lowp else op.aty(Y)

    Vk = None
    restart = 0
    while True:
        Vall = torch.empty((d, m_cap), dtype=torch.float32, device=dev)
        Bmat = torch.zeros((m_cap, m_cap), dtype=f64, device=dev)
        Vall[:, :b] = V0
        m = b                                  # columns of Vall in use
        Y = _av(_pad(Vall[:, :b], P))
        info.passes += 1
        info.lowp_passes += int(lowp)
        U, R = _cholqr2(op, Y, b)              # U: n x P (cols >= b are zero)
        Bmat[:b, :b] = R
        blocks = [(0, b)]                      # column ranges of the blocks
        Ublocks = None if (polish or lowp) else [U[:, :b].clone()]   # left Lanczos blocks (only needed without the polish)
        prev_res, prev_prev, stagn = None, None, 0
        done = False
        target = lowp_tol if lowp else tol
        while True:
            j0, j1 = blocks[-1]
            bj = j1 - j0
            # ---- would the next pass only CONFIRM convergence?  After a left update the Ritz triplets of the
            # current spaces are known without another pass (A V = U B exactly), only their right residual is not;
            # when the residual history predicts convergence, estimate it on 1/16 of the peaks (op.residual_sample)
            # and finish if the estimate is at most tol/2 (the estimator's spread over 1/16 of 200k peaks is a few %).  Otherwise (or if the operator cannot sample)
            # carry on with the full pass, which then decides as before.
            if (not lowp and Ublocks is not None and len(blocks) >= 2 and prev_res is not None and sample_check
                    and prev_res * min(prev_res / prev_prev if prev_prev else 0.1, 0.1) <= 3.0 * tol
                    and hasattr(op, "residual_sample")):
                with phase("lsi.ritz_svd"):
                    Bm = Bmat[:m, :m]
                    lam, Zr = torch.linalg.eigh(Bm.T @ Bm)
                    kk = min(k, m)
                    sig = lam.flip(0).clamp_min(0).sqrt()
                    Zt = Zr.flip(1).T.contiguous()
                    Vk_try = Vall[:, :m] @ Zt[:kk, :].T.to(torch.float32)
                    Xl = (Bm @ Zt[:kk, :].T) / sig[:kk].clamp_min(1e-300)
                    Uk_try = _pad(torch.cat(Ublocks, 1) @ Xl.to(torch.float32), P)
                est = op.residual_sample(Uk_try, Vk_try, sig[:kk])
                if _dist.is_distributed():
                    est = _dist.all_reduce_max_(est.contiguous())
                info.sampled_checks += 1
                if float(est.max()) <= tol / 2.0:
                    rmax = float(est.max())
                    info.history.append(rmax)
                    info.residuals = est.tolist()
                    info.sampled_stop = True
                    Vk, Uk_lanczos, s_lanczos = Vk_try, Uk_try[:, :kk].contiguous(), sig[:kk].clone()
                    V0_next = Vk
                    done = True
                    break
            # ---- right side: W = A^T U_j - V_j R_j^T, full reorth, QR --------------------
            W = _aty(U)[:, :bj].clone()
            info.passes += 1
            info.lowp_passes += int(lowp)
            with phase("lsi.reorth"):
                W -= Vall[:, j0:j1] @ Bmat[j0:j1, j0:j1].T.to(torch.float32)
                W, _ = _orth_against(W, Vall[:, :m])
            bn = min(bj, m_cap - m, d - m)     # width of the next block
            Sj = None
            if d - m > 0:
              with phase("lsi.qr"):
                Qn, S1 = _qr_dspace(op, W, P)
                # rank-deficient W leaves arbitrary directions in Qn: clean them against the basis
                Qn, _ = _orth_against(Qn.contiguous(), Vall[:, :m], passes=1)
                Qn, S2 = _qr_dspace(op, Qn, P)
                Sj = (S2.to(f64) @ S1.to(f64))          # W = Qn Sj   (bj x bj)
            # ---- Rayleigh-Ritz on the block-bidiagonal B (fp64, tiny) ---------------------
            with phase("lsi.ritz_svd"):
                # Ritz triplets of the block-bidiagonal B through eigh(B^T B) in fp64 (several times cheaper
                # than a full SVD; the squared condition number is harmless at 1e-16).  Only the last block
                # row of the left vectors is needed for the residuals: X = B Z / sigma.
                Bm = Bmat[:m, :m]
                lam, Zr = torch.linalg.eigh(Bm.T @ Bm)
                kk = min(k, m)
                sig = lam.flip(0).clamp_min(0).sqrt()
                Zt = Zr.flip(1).T.contiguous()
                Xlast = (Bm[j0:j1, :] @ Zt[:kk, :].T) / sig[:kk].clamp_min(1e-300)
            if Sj is not None:
                res = torch.linalg.norm(Sj @ Xlast, dim=0) / sig[:kk].clamp_min(1e-300)
            else:
                res = torch.zeros(kk, dtype=f64, device=dev)
            if _dist.is_distributed():
                # The d-space basis is REPLICATED: every rank ran the same library calls on bit-identical input (the
                # allreduced W), so Qn / Sj / res agree bit for bit without being exchanged.  One small MAX-allreduce
                # carries both the stopping decision (control flow must not diverge) and a fingerprint of the new
                # block that proves the replicas agree; only if they do not (never observed) rank 0's block is
                # broadcast.  Round 1 broadcast Qn (51 MB), Sj and res every step: three sync points, now one.
                if Sj is not None:
                    chk = (Qn.sum(dtype=f64) + Sj.sum()).reshape(1)
                else:
                    chk = torch.zeros(1, dtype=f64, device=dev)
                pack = _dist.all_reduce_max_(torch.cat([res, chk, -chk]))
                res = pack[:kk]
                if bool(pack[kk] != -pack[kk + 1]):
                    info.replica_repairs += 1
                    Qn = _dist.broadcast_(Qn.contiguous())
                    Sj = _dist.broadcast_(Sj.contiguous())
                    res = _dist.broadcast_((torch.linalg.norm(Sj @ Xlast, dim=0) / sig[:kk].clamp_min(1e-300)).contiguous())
            rmax = float(res.max())
            info.iterations += 1
            info.history.append(rmax)
            if verbose:
                print(f"[lsi] restart {restart} iter {info.iterations} basis {m} max rel residual {rmax:.3e}")
            if prev_res is not None and rmax > 0.5 * prev_res and rmax < 1e-3:
                stagn += 1
            else:
                stagn = 0
            prev_prev, prev_res = prev_res, rmax
            if rmax <= target or stagn >= 2 or bn <= 0:
                done = (rmax <= target) or stagn >= 2 or m >= d
                info.residuals = res.tolist()
                with phase("lsi.ritz_vectors"):
                    Vk = Vall[:, :m] @ Zt[:kk, :].T.to(torch.float32)      # d x k right Ritz vectors
                    V0_next = Vall[:, :m] @ Zt[:b, :].T.to(torch.float32)
                    if Ublocks is not None:                                # left Ritz vectors: U_all (B Z / sigma)
                        Xl = (Bm @ Zt[:kk, :].T) / sig[:kk].clamp_min(1e-300)
                        Uk_lanczos = torch.cat(Ublocks, 1) @ Xl.to(torch.float32)
                        s_lanczos = sig[:kk].clone()
                break
            # ---- left side: Y = A V_{j+1} - U_j S_j^T, CholeskyQR2 --------------------------
            Sj_use = Sj[:bn, :]                                    # if the block shrank keep bn rows
            Vall[:, m:m + bn] = Qn[:, :bn]
            Y = _av(_pad(Vall[:, m:m + bn], P))
            info.passes += 1
            info.lowp_passes += int(lowp)
            with phase("lsi.left_update"):
                M = torch.zeros((P, P), dtype=torch.float32, device=dev)
                M[:bj, :bn] = Sj_use.T.to(torch.float32)
                Y -= U @ M
            U, Rn = _cholqr2(op, Y, bn)
            Bmat[j0:j1, m:m + bn] = Sj_use.T
            Bmat[m:m + bn, m:m + bn] = Rn
            blocks.append((m, m + bn))
            if Ublocks is not None:
                Ublocks.append(U[:, :bn].clone())
            m += bn
        if lowp:
            # half-precision phase over: continue in fp32 from its Ritz vectors (not counted as a restart)
            lowp = False
            V0, _ = torch.linalg.qr(V0_next)
            continue
        info.basis = m
        info.converged = (rmax <= tol) or m >= d
        info.stalled = done and not info.converged
        if done or restart == max_restarts:
            break
        restart += 1
        info.restarts += 1
        V0, _ = torch.linalg.qr(V0_next)

    if not polish:
        return Uk_lanczos, s_lanczos, Vk, info
    # ---- final Rayleigh-Ritz polish, as scipy does after ARPACK (_svds.py:508-533) -------------
    with phase("lsi.final"):
        Vk, _ = _qr_dspace(op, Vk, P)
        Vk = Vk.contiguous()
        kk = Vk.shape[1]
        Y = op.av(_pad(Vk, P))
        info.passes += 1
        G = op.gram(Y, kk)
        lam, Z = torch.linalg.eigh(0.5 * (G + G.T))
        lam, Z = lam.flip(0), Z.flip(1)
        s = lam.clamp_min(0).sqrt()
        Zs = (Z / s.clamp_min(1e-300)).to(torch.float32)
        Mz = torch.zeros((P, kk), dtype=torch.float32, device=dev)
        Mz[:kk, :] = Zs
        Uk = Y @ Mz
        Vk = Vk @ Z.to(torch.float32)
    return Uk, s, Vk, info
