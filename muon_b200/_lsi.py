"""Truncated SVD driver for LSI: block Golub-Kahan-Lanczos with Rayleigh-Ritz.

The reference computes ``svds(adata.X, k)`` (muon/_atac/tools.py:53): ARPACK ``eigsh`` on the
implicit X^T X, one vector at a time -- 300-900 single-vector passes over the matrix for
k=50 (SURVEY section 6).  On an H100 every pass streams the whole CSR from HBM, so the design
goal is *few, wide* passes: a block of ``b`` vectors (b = padded kernel width, 64 for k=50)
per pass and a Krylov method that converges in a handful of block steps.

Algorithm (host side, all heavy work in the operator callbacks):

  V_1 = orth(randn(d, b));  U_1 R_1 = qr(A V_1)
  repeat   W = A^T U_j - V_j R_j^T                     (SpMM on A^T; allreduce over cell shards)
           W -= V_all (V_all^T W)   (x2)               (full reorthogonalisation, d-space, replicated)
           V_{j+1} S_j = qr(W)
           Y = A V_{j+1} - U_j S_j^T                   (SpMM on A; local to the cell shard)
           U_{j+1} R_{j+1} = cholqr2(Y)                (Gram kernel + b x b allreduce)
           B = blockbidiag(R, S^T);  svd(B) in fp64 -> Ritz values, residuals ||S_j x_last||
  until the first k residuals are below tol * sigma_i (or stagnate at the fp32 floor)
  V_k = V_all Z[:, :k];  U_k = U_all B Z[:, :k] / sigma        (A V_all = U_all B holds exactly)

Working on A (not A^T A) keeps the attainable accuracy at eps*sigma_1/sigma_i instead of
eps*(sigma_1/sigma_i)^2.  Reading U_k off the stored left blocks saves the extra pass over A that
scipy's Rayleigh-Ritz tail (``eigvec -> Av -> svd(Av)``, scipy _svds.py:508-533) spends; at the
tolerance used it does not change the result.

The driver is backend-agnostic: ``op`` supplies the products (protocol in ``truncated_svd``).  The
product wires the CUDA kernels (``CsrOperator``); CPU tests of this host logic inject a scipy
operator of their own.
"""
from __future__ import annotations

import functools
from dataclasses import dataclass, field
from typing import NamedTuple, Optional

import torch

from . import _dist
from ._lib import phase

LOWP_TOL = 1e-3     # target of the half-precision cycle: rounding the operand to half caps the residual near 2e-4


@dataclass
class SvdInfo:
    passes: int = 0              # sparse passes over A or A^T
    lowp_passes: int = 0         # of which with the dense operand rounded to IEEE half
    replica_repairs: int = 0     # multi-GPU: times the replicated d-space block had to be re-broadcast (expected 0)
    sampled_checks: int = 0      # residual estimates on 1/16 of the peaks (each costs 1/16 of a pass)
    sampled_stop: bool = False   # convergence was accepted on such an estimate (<= tol/2) instead of a full pass
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
            self.At = A.transpose_panels(pad)
        self.n_local, self.d = A.shape
        self.n_total = A.n_total
        self.device = A.data.device

    lowp = True      # av / aty accept lowp=True: dense operand rounded to IEEE half (csrc/spmm.cu)

    def av(self, V, lowp: bool = False):
        with phase("lsi.spmm_av"):
            return self._dev.spmm(self.A, self._dev.to_half_scaled(V) if lowp else V, dynamic=False)

    def aty(self, Y, lowp: bool = False):
        """A^T Y summed over the cell shards."""
        with phase("lsi.spmm_aty"):
            return _dist.all_reduce_sum_(self.At.spmm(Y, dynamic=True, half=lowp))

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


def _chol_upper_checked(G: torch.Tensor) -> Optional[torch.Tensor]:
    """Upper Cholesky factor of an fp64 Gram, or None if the block is too ill-conditioned for CholeskyQR in fp32."""
    G = 0.5 * (G + G.T)
    L, info = torch.linalg.cholesky_ex(G)
    dg = torch.diagonal(L)
    if int(info) != 0 or float(dg.min()) < 1e-4 * float(dg.max()):   # cond(W) > ~1e4: not safe in fp32
        return None
    return L.T


def _cholqr2(gram, Y: torch.Tensor, l: int, factor):
    """CholeskyQR2 of Y[rows x P] (first l columns meaningful; Gram ``gram(Y, l)``, upper factor ``factor(G)``) ->
    Q (same layout) and R[l x l] fp64, or None if ``factor`` refuses a Gram."""
    R_tot = None
    for _ in range(2):
        R = factor(gram(Y, l))
        if R is None:
            return None
        Rinv = torch.linalg.solve_triangular(R, torch.eye(l, dtype=R.dtype, device=R.device), upper=True)
        M = torch.zeros((Y.shape[1], Y.shape[1]), dtype=torch.float32, device=Y.device)
        M[:l, :l] = Rinv.to(torch.float32)
        Y = Y @ M
        R_tot = R if R_tot is None else R @ R_tot
    return Y, R_tot


def _qr_dspace(gram_local, W: torch.Tensor, P: int):
    """Thin QR of a replicated d x b block.  CholeskyQR2 on the operator's local Gram kernel when it has
    one and the block is well conditioned (0.3 ms instead of ~5 ms of Householder panels for
    200k x 64); Householder (cuSOLVER geqrf) otherwise."""
    l = W.shape[1]
    if gram_local is not None and l <= P and W.shape[0] >= 4 * l:
        qr = _cholqr2(gram_local, _pad(W, P), l, _chol_upper_checked)
        if qr is not None:
            return qr[0][:, :l], qr[1].to(torch.float32)
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


def _ritz(Bm: torch.Tensor):
    """Ritz values (descending) and Z^T of the block-bidiagonal B through eigh(B^T B) in fp64 (several times
    cheaper than a full SVD; the squared condition number is harmless at 1e-16)."""
    lam, Zr = torch.linalg.eigh(Bm.T @ Bm)
    return lam.flip(0).clamp_min(0).sqrt(), Zr.flip(1).T.contiguous()


def _left_ritz(Ublocks, Bm, sig, Zt, k):
    """The k left Ritz vectors U_all (B Z / sigma) from the stored left Lanczos blocks."""
    return torch.cat(Ublocks, 1) @ ((Bm @ Zt[:k, :].T) / sig[:k].clamp_min(1e-300)).to(torch.float32)


class _Cycle(NamedTuple):
    s: torch.Tensor                 # k Ritz values, descending, fp64
    V: torch.Tensor                 # d x k right Ritz vectors
    U: Optional[torch.Tensor]       # n_local x k left Ritz vectors; None if the cycle kept no left blocks
    V0_next: torch.Tensor           # d x b restart block (the top b Ritz vectors, not re-orthonormalised)
    rmax: float                     # largest relative residual of the k triplets
    m: int                          # basis size
    done: bool                      # stopped for good: converged, stagnated, or the basis is the whole space


def _cycle(op, V0, tol, *, k, P, m_cap, info, lowp, gram_local, sample, verbose):
    """One block Golub-Kahan cycle from the orthonormal start block V0 [d x b].

    Runs until the k wanted triplets reach relative residual ``tol``, the residuals stagnate, or the basis reaches
    ``m_cap`` columns.  With ``lowp`` every product takes its dense operand rounded to IEEE half and no left blocks
    are kept.  Otherwise the left Lanczos blocks are kept for U_k, and ``sample`` (the operator's
    ``residual_sample``, or None) may end the cycle on a residual estimate instead of a pass over A^T.  Passes,
    iterations and residuals are counted into ``info``."""
    d, dev, f64 = op.d, op.device, torch.float64
    b = V0.shape[1]

    def av(V):
        info.passes += 1
        info.lowp_passes += int(lowp)
        return op.av(V, lowp=True) if lowp else op.av(V)

    def aty(Y):
        info.passes += 1
        info.lowp_passes += int(lowp)
        return op.aty(Y, lowp=True) if lowp else op.aty(Y)

    Vall = torch.empty((d, m_cap), dtype=torch.float32, device=dev)
    Bmat = torch.zeros((m_cap, m_cap), dtype=f64, device=dev)
    Vall[:, :b] = V0
    m = b                                  # columns of Vall in use
    j0, j1 = 0, b                          # columns of the newest block
    Y = av(_pad(Vall[:, :b], P))
    with phase("lsi.cholqr"):
        U, R = _cholqr2(op.gram, Y, b, _chol_upper)          # U: n x P (cols >= b are zero)
    Bmat[:b, :b] = R
    Ublocks = None if lowp else [U[:, :b].clone()]          # left Lanczos blocks
    prev_res, prev_prev, stagn = None, None, 0
    while True:
        bj = j1 - j0
        ritz = None
        # ---- would the next pass only CONFIRM convergence?  After a left update the Ritz triplets of the
        # current spaces are known without another pass (A V = U B exactly), only their right residual is not;
        # when the residual history predicts convergence, estimate it on 1/16 of the peaks (op.residual_sample)
        # and finish if the estimate is at most tol/2 (the estimator's spread over 1/16 of 200k peaks is a few %).
        # Otherwise carry on with the full pass, which then decides as before.
        if (sample is not None and Ublocks is not None and prev_res is not None
                and prev_res * min(prev_res / prev_prev if prev_prev else 0.1, 0.1) <= 3.0 * tol):
            with phase("lsi.ritz_svd"):
                Bm = Bmat[:m, :m]
                ritz = _ritz(Bm)
                sig, Zt = ritz
                Vk = Vall[:, :m] @ Zt[:k, :].T.to(torch.float32)
                Uk = _left_ritz(Ublocks, Bm, sig, Zt, k)
            est = sample(_pad(Uk, P), Vk, sig[:k])
            if _dist.is_distributed():
                est = _dist.all_reduce_max_(est.contiguous())
            info.sampled_checks += 1
            if float(est.max()) <= tol / 2.0:
                rmax = float(est.max())
                info.history.append(rmax)
                info.residuals = est.tolist()
                info.sampled_stop = True
                return _Cycle(sig[:k].clone(), Vk, Uk, Vk, rmax, m, True)
        # ---- right side: W = A^T U_j - V_j R_j^T, full reorth, QR --------------------
        W = aty(U)[:, :bj].clone()
        with phase("lsi.reorth"):
            W -= Vall[:, j0:j1] @ Bmat[j0:j1, j0:j1].T.to(torch.float32)
            W, _ = _orth_against(W, Vall[:, :m])
        bn = min(bj, m_cap - m, d - m)     # width of the next block
        Sj = None
        if d - m > 0:
            with phase("lsi.qr"):
                Qn, S1 = _qr_dspace(gram_local, W, P)
                # rank-deficient W leaves arbitrary directions in Qn: clean them against the basis
                Qn, _ = _orth_against(Qn.contiguous(), Vall[:, :m], passes=1)
                Qn, S2 = _qr_dspace(gram_local, Qn, P)
                Sj = (S2.to(f64) @ S1.to(f64))          # W = Qn Sj   (bj x bj)
        # ---- Rayleigh-Ritz on the block-bidiagonal B (fp64, tiny) ---------------------
        with phase("lsi.ritz_svd"):
            # Only the last block row of the left vectors is needed for the residuals: X = B Z / sigma.
            Bm = Bmat[:m, :m]
            if ritz is None:                   # else the sampled check has decomposed this same B
                ritz = _ritz(Bm)
            sig, Zt = ritz
            Xlast = (Bm[j0:j1, :] @ Zt[:k, :].T) / sig[:k].clamp_min(1e-300)
        if Sj is not None:
            res = torch.linalg.norm(Sj @ Xlast, dim=0) / sig[:k].clamp_min(1e-300)
        else:
            res = torch.zeros(k, dtype=f64, device=dev)
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
            res = pack[:k]
            if bool(pack[k] != -pack[k + 1]):
                info.replica_repairs += 1
                Qn = _dist.broadcast_(Qn.contiguous())
                Sj = _dist.broadcast_(Sj.contiguous())
                res = _dist.broadcast_((torch.linalg.norm(Sj @ Xlast, dim=0) / sig[:k].clamp_min(1e-300)).contiguous())
        rmax = float(res.max())
        info.iterations += 1
        info.history.append(rmax)
        if verbose:
            print(f"[lsi] restart {info.restarts} iter {info.iterations} basis {m} max rel residual {rmax:.3e}")
        if prev_res is not None and rmax > 0.5 * prev_res and rmax < 1e-3:
            stagn += 1
        else:
            stagn = 0
        prev_prev, prev_res = prev_res, rmax
        if rmax <= tol or stagn >= 2 or bn <= 0:
            info.residuals = res.tolist()
            with phase("lsi.ritz_vectors"):
                Vk = Vall[:, :m] @ Zt[:k, :].T.to(torch.float32)       # d x k right Ritz vectors
                V0_next = Vall[:, :m] @ Zt[:b, :].T.to(torch.float32)
                Uk = None if Ublocks is None else _left_ritz(Ublocks, Bm, sig, Zt, k)
            return _Cycle(sig[:k].clone(), Vk, Uk, V0_next, rmax, m, rmax <= tol or stagn >= 2 or m >= d)
        # ---- left side: Y = A V_{j+1} - U_j S_j^T, CholeskyQR2 --------------------------
        Sj_use = Sj[:bn, :]                                    # if the block shrank keep bn rows
        Vall[:, m:m + bn] = Qn[:, :bn]
        Y = av(_pad(Vall[:, m:m + bn], P))
        with phase("lsi.left_update"):
            M = torch.zeros((P, P), dtype=torch.float32, device=dev)
            M[:bj, :bn] = Sj_use.T.to(torch.float32)
            Y -= U @ M
        with phase("lsi.cholqr"):
            U, Rn = _cholqr2(op.gram, Y, bn, _chol_upper)
        Bmat[j0:j1, m:m + bn] = Sj_use.T
        Bmat[m:m + bn, m:m + bn] = Rn
        if Ublocks is not None:
            Ublocks.append(U[:, :bn].clone())
        j0, j1 = m, m + bn
        m += bn


def truncated_svd(op, k: int, pad_to: int, tol: float = 1e-5, max_basis: Optional[int] = None,
                  max_restarts: int = 4, seed: int = 0, verbose: bool = False):
    """Top-k singular triplets of the (cell-sharded) matrix behind ``op``.

    Returns (U [n_local x k] fp32, s [k] fp64, V [d x k] fp32, SvdInfo).  ``pad_to`` is the padded
    dense width P the kernels run at (32/64/128); the Krylov block size is min(P, d, n_total).

    ``op`` provides ``d`` (columns of A), ``device`` and
      ``av(V)``        A V [n_local x P] for V [d x P];
      ``aty(Y)``       A^T Y [d x P] for Y [n_local x P], summed over the cell shards;
      ``gram(Y, l)``   Y[:, :l]^T Y[:, :l] [l x l] in fp64, summed over the cell shards;
    and optionally
      ``n_total``                       rows of A over all shards (caps the block size);
      ``lowp``                          true if ``av`` and ``aty`` accept ``lowp=True``: the dense operand rounded
                                        to IEEE half;
      ``gram_local(Y, l)``              ``gram`` without the sum over shards, for CholeskyQR2 of the replicated
                                        d-space blocks (Householder QR without it);
      ``residual_sample(Uk, Vk, sig)``  an estimate of the relative residuals ||A^T u_i - sigma_i v_i|| / sigma_i
                                        of k triplets, from a sample of the rows of A^T.

    Schedule: if the operator has ``lowp`` and ``tol`` < LOWP_TOL, a first cycle runs with the dense operand of
    every product rounded to half -- half the bytes through the gather path that bounds the SpMM kernel -- until
    the wanted triplets reach LOWP_TOL; it does not count as a restart.  Then fp32 cycles run from the Ritz
    vectors of the previous one, restarting up to ``max_restarts`` times: one fp32 block step takes residuals
    from ~3e-4 to below 1e-5.  ``SvdInfo.lowp_passes`` counts the half-precision passes.  When the residual
    history predicts that the next pass over A^T would only confirm convergence and the operator has
    ``residual_sample``, the residuals are first estimated on that sample, and the cycle stops if the estimate
    is <= tol/2; the full pass is skipped only then.  U_k is read off the stored left Lanczos blocks.
    """
    d, dev, P = op.d, op.device, pad_to
    lowp = bool(getattr(op, "lowp", False)) and tol < LOWP_TOL
    gram_local = getattr(op, "gram_local", None)
    sample = getattr(op, "residual_sample", None)
    k = int(k)
    b = min(P, d, getattr(op, "n_total", d))
    assert 1 <= k <= b, (k, b)
    m_cap = min(d, max_basis if max_basis is not None else 16 * P)
    m_cap = max(m_cap, min(d, 2 * b))
    info = SvdInfo(block=b)
    cycle = functools.partial(_cycle, op, k=k, P=P, m_cap=m_cap, info=info, gram_local=gram_local,
                              sample=sample, verbose=verbose)

    with phase("lsi.init"):
        g = torch.Generator(device=dev).manual_seed(int(seed))   # same stream on every rank (same device type)
        V0 = torch.randn((d, b), generator=g, dtype=torch.float32, device=dev)
        V0, _ = _qr_dspace(gram_local, V0, P)

    if lowp:
        V0, _ = torch.linalg.qr(cycle(V0, LOWP_TOL, lowp=True).V0_next)
    while True:
        c = cycle(V0, tol, lowp=False)
        info.basis = c.m
        info.converged = c.rmax <= tol or c.m >= d
        info.stalled = c.done and not info.converged
        if c.done or info.restarts == max_restarts:
            return c.U, c.s, c.V, info
        info.restarts += 1
        V0, _ = torch.linalg.qr(c.V0_next)
