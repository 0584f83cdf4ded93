"""``mu.tl.mofa`` on the GPU: MOFA+ coordinate-ascent VI over sparse, implicitly-centred modalities.

Reference: ``muon._core.tools.mofa`` (muon/_core/tools.py:290-708) marshals the MuData into dense
arrays (tools.py:117-141), trains mofapy2 (tools.py:583-585) and copies E[Z], E[W] and the variance
explained into ``obsm["X_mofa"]``, ``varm["LFs"]``, ``uns["mofa"]`` (tools.py:604-701).

Here the modalities stay sparse in HBM.  Per iteration and view there are exactly two passes over
the data -- ``P = Y^T E[Z]`` and ``Q = Y (tau * E[W])``, both the CSR SpMM kernel -- plus fused
per-row Gauss-Seidel kernels (csrc/mofa.cu) and K x K statistics from the Gram kernel.  Cells are
sharded across ranks; ``P``, the K x K Gram and K-vectors are sum-allreduced (SURVEY section 8e).
The update equations and their order are those of oracle/mofa_ref.py (see its header for the
parity status against mofapy2).

Supported: gaussian views kept sparse (implicit centring), poisson / bernoulli views as dense Seeger pseudo-data
(guessed from the data like mofapy2 does when ``likelihoods=None``), ``groups_label``, ``use_obs`` union /
intersection (cells missing from whole views), ``use_var`` feature subsets, ``use_layer``, ``scale_views``,
``scale_groups``, ``center_groups``, ARD on weights / factors, spike-and-slab weights, convergence modes, ``copy``;
the one-group case also cell-sharded over several GPUs.  Not supported (``NotImplementedError``, never a silent
substitute): ``spikeslab_factors``, ``use_raw``, SVI, MEFISTO smoothing; ``outfile`` (HDF5) is ignored (h5py is not
available); ``n_factors`` > 64.
"""
from __future__ import annotations

from functools import reduce
from typing import Optional
from warnings import warn

import numpy as np
import torch

from . import _device, _dist
from ._containers import SimpleMuData, is_anndata, is_mudata
from ._lib import call, ptr, stream_ptr

A0 = B0 = 1e-3
TH_A0 = TH_B0 = 1.0
TOLERANCE = {"fast": 5e-4, "medium": 5e-5, "slow": 5e-6}
f64 = torch.float64


class _Block:
    """One (view, group) block: the cells of group g observed in view m, as a compact CSR with its
    transpose panels, plus where those cells sit in the local factor matrix."""

    def __init__(self, A: _device.DeviceCSR, rows, lo: int, hi: int, ld: int):
        self.A, self.At = A, A.transpose_panels(ld)
        self.rows, self.lo, self.hi = rows, lo, hi      # rows: LongTensor into local Z, or None = Z[lo:hi]
        self.n_local = A.shape[0]

    def take(self, Z):                                   # rows of Z belonging to this block (contiguous n x ld)
        return Z[self.lo:self.hi] if self.rows is None else Z.index_select(0, self.rows)

    def aty(self, Zb):                                   # Y_b^T Z_b  (D x ld): transposed sparse pass
        return self.At.spmm(Zb.contiguous(), dynamic=True)

    def add_av(self, Q, tw):                             # Q[rows of the block] += Y_b (tau * W)
        if self.rows is None:
            _device.spmm(self.A, tw, out=Q[self.lo:self.hi], accumulate=True, dynamic=False)
        else:
            Q.index_add_(0, self.rows, _device.spmm(self.A, tw, dynamic=False))

    def moments(self, D, dev):
        """per-feature sum and sum of squares over the block's cells (fp64), from the transposed panels"""
        s1, s2 = torch.zeros(D, dtype=f64, device=dev), torch.zeros(D, dtype=f64, device=dev)
        self.At.wait()
        for (_, _, T) in self.At.panels:
            t1, t2 = torch.empty(D, dtype=f64, device=dev), torch.empty(D, dtype=f64, device=dev)
            if isinstance(T, _device.DevicePairs):
                call("mub_csrp_row_stats_f32", ptr(T.indptr), ptr(T.pairs), D, ptr(t1), ptr(t2), stream_ptr())
            else:
                call("mub_csr_row_stats_f32", ptr(T.indptr), ptr(T.data), D, ptr(t1), ptr(t2), stream_ptr())
            s1 += t1
            s2 += t2
        return s1, s2


class _DenseBlock:
    """One (view, group) block of a NON-gaussian view: the observations as a dense row-major fp32 matrix and the
    Seeger pseudo-data that stand in for them (dense by construction: zeta = E[Z] E[W]^T is).  The contractions
    are GEMMs (cuBLAS via torch); the elementwise passes are csrc/mofa_pseudo.cu."""

    def __init__(self, obs: torch.Tensor, rows, lo: int, hi: int):
        assert obs.dtype == torch.float32 and obs.is_contiguous() and obs.dim() == 2
        self.obs, self.Y = obs, torch.zeros_like(obs)
        self.rows, self.lo, self.hi = rows, lo, hi
        self.n_local = obs.shape[0]

    def take(self, Z):
        return Z[self.lo:self.hi] if self.rows is None else Z.index_select(0, self.rows)

    def aty(self, Zb):
        return self.Y.T @ Zb

    def add_av(self, Q, tw):
        if self.rows is None:
            Q[self.lo:self.hi].addmm_(self.Y, tw)
        else:
            Q.index_add_(0, self.rows, self.Y @ tw)


class _View:
    """One modality: blocks per group, per-(group, feature) moments, variational state of W / alpha / theta / tau."""

    def __init__(self, blocks, D: int, K: int, ld: int, center: bool, scale_views: bool, scale_groups: bool, dev,
                 lik: str = "gaussian"):
        self.blocks, self.D, self.G = blocks, D, len(blocks)
        self.lik = lik
        self.kind = {"gaussian": 0, "poisson": 1, "bernoulli": 2}[lik]
        G = self.G
        s1 = torch.zeros((G, D), dtype=f64, device=dev)
        s2 = torch.zeros((G, D), dtype=f64, device=dev)
        cnt = torch.zeros(G, dtype=f64, device=dev)
        mx = torch.zeros(D, dtype=torch.float32, device=dev)
        for g, b in enumerate(blocks):
            cnt[g] = b.n_local
            if b.n_local == 0:
                continue
            if self.kind == 0:
                s1[g], s2[g] = b.moments(D, dev)
            else:
                mx = torch.maximum(mx, b.obs.max(0).values)
        if self.kind != 0:
            # non-gaussian view: no centring, no scaling, precision fixed at Seeger's bound (oracle/mofa_ref.py)
            _dist.all_reduce_sum_(cnt)
            _dist.all_reduce_max_(mx)
            self.n = cnt
            self.mean = torch.zeros((G, D), dtype=f64, device=dev)
            self.mu32, self.mu64 = None, self.mean
            self.inv_scale = torch.ones(G, dtype=f64, device=dev)
            self.ssq = torch.zeros((G, D), dtype=f64, device=dev)          # of the pseudo-data: refreshed every iteration
            kappa = (0.25 + 0.17 * mx.to(f64)) if self.kind == 1 else torch.full((D,), 0.25, dtype=f64, device=dev)
            self.kappa32 = kappa.to(torch.float32).contiguous()
            self._init_state(K, ld, dev)
            self.tau = (kappa[None, :].expand(G, D).contiguous(), torch.ones((G, D), dtype=f64, device=dev))
            return
        _dist.all_reduce_sum_(s1)
        _dist.all_reduce_sum_(s2)
        _dist.all_reduce_sum_(cnt)
        self.n = cnt                                                # cells per group observed in this view (global)
        nn = cnt.clamp_min(1.0)[:, None]
        self.mean = s1 / nn                                        # intercepts per group, tools.py:283-286
        # center_groups=False still centres every feature, with its mean over ALL groups (mofapy2 process_data,
        # [recalled]); with a single group the flag therefore changes nothing
        mu = self.mean if center else (s1.sum(0) / cnt.sum().clamp_min(1.0))[None, :].expand(G, D).contiguous()
        center = True
        ssq = (s2 - 2.0 * mu * s1 + cnt[:, None] * mu * mu).clamp_min(0)      # sum_n (y - mu)^2 per (g, d)
        tot = s1 - cnt[:, None] * mu                               # sum_n (y - mu)
        self.mu32 = mu.to(torch.float32).contiguous() if center else None
        self.mu64 = mu
        inv = torch.ones(G, dtype=f64, device=dev)
        if scale_views:                                            # global std of the (centred) view
            nel = cnt.sum() * D
            var = ssq.sum() / nel - (tot.sum() / nel) ** 2
            inv[:] = 1.0 / torch.sqrt(var) if float(var) > 0 else 1.0
        if scale_groups:                                           # per-group std (takes precedence)
            nel = (cnt * D).clamp_min(1.0)
            var = ssq.sum(1) / nel - (tot.sum(1) / nel) ** 2
            inv = torch.where(var > 0, 1.0 / torch.sqrt(var.clamp_min(1e-300)), torch.ones_like(var))
        self.inv_scale = inv.contiguous()
        self.ssq = (ssq * (inv ** 2)[:, None]).contiguous()
        self._init_state(K, ld, dev)

    def _init_state(self, K, ld, dev):
        D, G = self.D, self.G
        z = lambda: torch.zeros((D, ld), dtype=torch.float32, device=dev)  # noqa: E731
        self.W, self.WW, self.S, self.What2 = z(), z(), z(), z()
        self.S[:, :K] = 1.0
        self.What2[:, :K] = 1.0
        one = lambda *sh: torch.ones(sh, dtype=f64, device=dev)    # noqa: E731
        self.alpha = (one(K), one(K))
        self.theta = (one(K), torch.full((K,), 1e-8, dtype=f64, device=dev))
        self.tau = (one(G, D), one(G, D))
        self.P = torch.zeros((G, D, ld), dtype=torch.float32, device=dev)   # Y^T E[Z] per group, un-centred
        self.ZZ = torch.zeros((G, K, K), dtype=f64, device=dev)            # E[Z^T Z] over the block's cells
        self.ZZ_mean = torch.zeros((G, K, K), dtype=f64, device=dev)
        self.zsum = torch.zeros((G, K), dtype=f64, device=dev)


def _E_gamma(ab):
    a, b = ab
    return a / b, torch.special.digamma(a) - torch.log(b)


def _E_beta(ab):
    a, b = ab
    dg = torch.special.digamma
    return dg(a) - dg(a + b), dg(b) - dg(a + b)


def _kl_gamma(ab, a0, b0):
    a, b = ab
    E, Eln = _E_gamma(ab)
    lg = torch.special.gammaln
    a0t, b0t = torch.tensor(a0, dtype=f64, device=a.device), torch.tensor(b0, dtype=f64, device=a.device)
    lp = a0t * torch.log(b0t) - lg(a0t) + (a0 - 1) * Eln - b0 * E
    lq = a * torch.log(b) - lg(a) + (a - 1) * Eln - b * E
    return float((lp - lq).sum())


def _kl_beta(ab, a0, b0):
    a, b = ab
    Eln, Eln1 = _E_beta(ab)
    lg = torch.special.gammaln
    c = float(lg(torch.tensor(a0 + b0, dtype=f64)) - lg(torch.tensor(a0, dtype=f64)) - lg(torch.tensor(b0, dtype=f64)))
    lp = c + (a0 - 1) * Eln + (b0 - 1) * Eln1
    lq = lg(a + b) - lg(a) - lg(b) + (a - 1) * Eln + (b - 1) * Eln1
    return float((lp - lq).sum())


class MofaDevice:
    """CAVI state machine on the device: gaussian views, G groups of cells, cells may be missing from
    whole views (the reference's ``use_obs="union"``), cell-sharded across ranks.

    ``blocks[m][g]`` = (DeviceCSR of the local cells of group g observed in view m, rows) where ``rows`` is a
    LongTensor of positions in the local factor matrix or a (lo, hi) range.  ``group_ranges[g]`` = (lo, hi) of
    group g in the local cell order (cells are ordered by group, as the reference does, tools.py:243-255);
    ``cls`` = int32 class id per local cell = g * 2^M + bitmask of the views it is observed in (None: all
    cells in class (0, all views)); ``n_groups_total[g]`` = global number of cells of group g.
    """

    def __init__(self, blocks, dims, group_ranges, n_groups_total, cls, K, Z0, center=True, scale_views=False,
                 scale_groups=False, ard_weights=True, ard_factors=True, spikeslab_weights=True, likelihoods=None):
        self.K = int(K)
        self.liks = ["gaussian"] * len(blocks) if likelihoods is None else list(likelihoods)
        if K > 64:
            raise NotImplementedError("n_factors > 64 is not supported yet")
        self.ld = ld = _device.pad_width(K)
        self.M, self.G = len(blocks), len(group_ranges)
        self.opts = (ard_weights, ard_factors, spikeslab_weights)
        dev = Z0.device if Z0.device.type == "cuda" else torch.device("cuda", torch.cuda.current_device())
        self.dev = dev
        self.group_ranges = group_ranges
        self.n_local = group_ranges[-1][1]
        self.Ng = torch.tensor([float(x) for x in n_groups_total], dtype=f64, device=dev)
        self.N = int(sum(n_groups_total))
        self.C = self.G << self.M
        # how many cells of class c each (view, group) block / each group holds (global): for sums of Var[z]
        if cls is None:                                   # every cell observed in every view
            cls = torch.empty(self.n_local, dtype=torch.int32, device=dev)
            for g, (lo, hi) in enumerate(group_ranges):
                cls[lo:hi] = (g << self.M) | ((1 << self.M) - 1)
        self.cls = cls
        counts = torch.bincount(cls.to(torch.int64), minlength=self.C).to(f64)
        self.class_count = _dist.all_reduce_sum_(counts)
        self.views = []
        for m in range(self.M):
            bl = []
            for g in range(self.G):
                A, rows = blocks[m][g]
                r, lo, hi = (None, rows[0], rows[1]) if isinstance(rows, tuple) else (rows, 0, 0)
                if self.liks[m] == "gaussian":
                    bl.append(_Block(A, r, lo, hi, ld))
                else:                                     # A: dense fp32 observations (n_b x D) on the device
                    bl.append(_DenseBlock(A, r, lo, hi))
            self.views.append(_View(bl, dims[m], K, ld, center, scale_views, scale_groups, dev, self.liks[m]))
        self.Z = torch.zeros((self.n_local, ld), dtype=torch.float32, device=dev)
        self.Z[:, :K] = Z0.to(dev, torch.float32)
        self.zvar = torch.ones((self.C, K), dtype=f64, device=dev)
        self.alphaZ = (torch.ones((self.G, K), dtype=f64, device=dev), torch.ones((self.G, K), dtype=f64, device=dev))
        self.elbo = []
        self._stats_Z()

    def _class_members(self, m, g):
        """class ids of group g whose cells are observed in view m"""
        return [(g << self.M) | bits for bits in range(1 << self.M) if bits & (1 << m)]

    # -- sufficient statistics of Z: one transposed sparse pass per (view, group) block + Grams -----------------
    def _stats_Z(self):
        K = self.K
        dK = torch.arange(K, device=self.dev)
        for m, v in enumerate(self.views):
            for g, b in enumerate(v.blocks):
                if b.n_local > 0:
                    Zb = b.take(self.Z)
                    ZZ = _device.gram(Zb, K, reduce=False)
                    zs = Zb[:, :K].sum(0, dtype=f64)
                    P = b.aty(Zb.contiguous())
                else:
                    ZZ = torch.zeros((K, K), dtype=f64, device=self.dev)
                    zs = torch.zeros(K, dtype=f64, device=self.dev)
                    P = torch.zeros((v.D, self.ld), dtype=torch.float32, device=self.dev)
                v.ZZ_mean[g], v.zsum[g], v.P[g] = ZZ, zs, P
            _dist.all_reduce_sum_(v.ZZ_mean)
            _dist.all_reduce_sum_(v.zsum)
            _dist.all_reduce_sum_(v.P)
            v.ZZ = v.ZZ_mean.clone()
            for g in range(self.G):
                cl = self._class_members(m, g)
                v.ZZ[g, dK, dK] += (self.class_count[cl, None] * self.zvar[cl]).sum(0)
        # E[z^2] summed over all cells of a group (for AlphaZ)
        ez2 = torch.zeros((self.G, K), dtype=f64, device=self.dev)
        for g, (lo, hi) in enumerate(self.group_ranges):
            if hi > lo:
                ez2[g] = (self.Z[lo:hi, :K].to(f64) ** 2).sum(0)
        _dist.all_reduce_sum_(ez2)
        for g in range(self.G):
            cl = list(range(g << self.M, (g + 1) << self.M))
            ez2[g] += (self.class_count[cl, None] * self.zvar[cl]).sum(0)
        self.Ez2 = ez2

    def step(self):
        K, ld, st, G, M, C = self.K, self.ld, stream_ptr(), self.G, self.M, self.C
        ard_w, ard_f, ss = self.opts
        onesK = torch.ones(K, dtype=f64, device=self.dev)
        # ---- Y: pseudo-data of the non-gaussian views (and the statistics that depend on them) -------------------
        for v in self.views:
            if v.kind != 0:
                self._pseudo(v)
        # ---- W ----------------------------------------------------------------------------------------
        for v in self.views:
            Etau = _E_gamma(v.tau)[0].to(torch.float32).contiguous()              # G x D
            Ea = (_E_gamma(v.alpha)[0] if ard_w else onesK).contiguous()
            lnth, ln1mth = _E_beta(v.theta)
            call("mub_mofa_update_w_f32", ptr(v.P), ptr(v.mu32), ptr(v.zsum), ptr(v.inv_scale), ptr(v.ZZ), ptr(Etau),
                 ptr(Ea), ptr(lnth.contiguous()), ptr(ln1mth.contiguous()), ptr(v.W), ptr(v.WW), ptr(v.S),
                 ptr(v.What2), v.D, ld, K, G, 1 if ss else 0, st)
            v.Etau32 = Etau
        # ---- Z ----------------------------------------------------------------------------------------
        Q = torch.zeros((self.n_local, ld), dtype=torch.float32, device=self.dev)
        GW = torch.zeros((C, K, K), dtype=f64, device=self.dev)
        cW = torch.zeros((C, K), dtype=f64, device=self.dev)
        qshift = torch.zeros((C, K), dtype=f64, device=self.dev)
        for m, v in enumerate(self.views):
            for g, b in enumerate(v.blocks):
                tw = (v.W * (v.Etau32[g] * v.inv_scale[g].to(torch.float32))[:, None]).contiguous()   # D x ld operand
                if b.n_local > 0:
                    b.add_av(Q, tw)
                qs = (v.mu64[g][:, None] * tw[:, :K].to(f64)).sum(0) if v.mu32 is not None else 0.0
                gw = _device.gram(v.W, K, weights=v.Etau32[g].contiguous(), reduce=False)
                cw = v.Etau32[g].to(f64) @ v.WW[:, :K].to(f64)
                for c in self._class_members(m, g):
                    GW[c] += gw
                    cW[c] += cw
                    qshift[c] += qs
        EaZ = _E_gamma(self.alphaZ)[0] if ard_f else torch.ones((G, K), dtype=f64, device=self.dev)
        self.zvar = (1.0 / (EaZ.repeat_interleave(1 << M, dim=0) + cW)).contiguous()
        call("mub_mofa_update_z_f32", ptr(Q), ptr(qshift.contiguous()), ptr(GW.contiguous()), ptr(self.zvar),
             ptr(self.cls), ptr(self.Z), self.n_local, ld, K, C, st)
        del Q
        self._stats_Z()
        # ---- AlphaW, ThetaW, AlphaZ ---------------------------------------------------------------------
        for v in self.views:
            if ard_w:
                v.alpha = (torch.full((K,), A0 + 0.5 * v.D, dtype=f64, device=self.dev),
                           B0 + 0.5 * v.What2[:, :K].sum(0, dtype=f64))
            if ss:
                s1 = v.S[:, :K].sum(0, dtype=f64)
                v.theta = (TH_A0 + s1, TH_B0 + v.D - s1)
        if ard_f:
            self.alphaZ = ((A0 + 0.5 * self.Ng)[:, None].expand(G, K).contiguous(), B0 + 0.5 * self.Ez2)
        # ---- Tau ----------------------------------------------------------------------------------------
        for v in self.views:
            if v.kind != 0:                                  # Seeger bound: the precision is a constant
                continue
            b = torch.empty((G, v.D), dtype=f64, device=self.dev)
            for g in range(G):
                call("mub_mofa_tau_f32", ptr(v.P[g]), ptr(v.mu32[g]) if v.mu32 is not None else None, ptr(v.zsum[g]),
                     float(v.inv_scale[g]), ptr(v.ZZ[g]), ptr(v.ssq[g]), ptr(v.W), ptr(v.WW), B0, ptr(b[g]), v.D, ld,
                     K, st)
            v.tau = ((A0 + 0.5 * v.n)[:, None].expand(G, v.D).contiguous(), b)
        self.elbo.append(self._elbo())

    def _pseudo(self, v):
        """Seeger pseudo-data of a non-gaussian view around zeta = E[Z] E[W]^T (csrc/mofa_pseudo.cu), then the
        statistics of the view that depend on them: P = Yhat^T E[Z] and sum Yhat^2 per feature."""
        K, st = self.K, stream_ptr()
        Wk = v.W[:, :K].contiguous()
        for g, b in enumerate(v.blocks):
            if b.n_local == 0:
                v.P[g].zero_()
                v.ssq[g].zero_()
                continue
            Zb = b.take(self.Z).contiguous()
            torch.matmul(Zb[:, :K], Wk.T, out=b.Y)
            call("mub_mofa_pseudo_f32", ptr(b.Y), ptr(b.obs), ptr(v.kappa32), b.n_local, v.D, v.kind, st)
            v.P[g] = b.aty(Zb)
            v.ssq[g] = (b.Y * b.Y).sum(0, dtype=f64)
        _dist.all_reduce_sum_(v.P)
        _dist.all_reduce_sum_(v.ssq)

    def _loglik(self, v):
        """sum over the observed entries of ln p(y | zeta) at zeta = E[Z] E[W]^T (the ELBO term of a non-gaussian view)"""
        K, st = self.K, stream_ptr()
        acc = torch.zeros(1, dtype=f64, device=self.dev)
        Wk = v.W[:, :K].contiguous()
        for b in v.blocks:
            if b.n_local == 0:
                continue
            zeta = b.take(self.Z)[:, :K].contiguous() @ Wk.T
            call("mub_mofa_loglik_f32", ptr(zeta), ptr(b.obs), b.n_local, v.D, v.kind, ptr(acc), st)
        return float(_dist.all_reduce_sum_(acc)[0])

    def _elbo(self):
        """Same expression as oracle/mofa_ref.py (tau trick; valid right after the Tau update)."""
        K, G, M = self.K, self.G, self.M
        ard_w, ard_f, ss = self.opts
        total = 0.0
        two_pi = 2.0 * np.pi
        for v in self.views:
            if v.kind == 0:
                Etau, Elntau = _E_gamma(v.tau)
                total += float((0.5 * v.n[:, None] * (Elntau - np.log(two_pi)) - Etau * (v.tau[1] - B0)).sum())
                total += _kl_gamma(v.tau, A0, B0)
            else:
                total += self._loglik(v)
            if ard_w:
                Ea, Elna = _E_gamma(v.alpha)
            else:
                Ea, Elna = torch.ones(K, dtype=f64, device=self.dev), torch.zeros(K, dtype=f64, device=self.dev)
            S0 = v.S[:, :K].to(f64)
            W, WW = v.W[:, :K].to(f64), v.WW[:, :K].to(f64)
            W2 = WW + (1.0 - S0) / Ea[None, :]     # spike branch at the current E[alpha] (see oracle/mofa_ref.py::elbo)
            S = S0.clamp(1e-300, 1.0)
            lp = -0.5 * np.log(two_pi) + 0.5 * Elna[None, :] - 0.5 * Ea[None, :] * W2
            Sd = S0.clamp_min(1e-300)
            var1 = torch.where(S0 > 0, WW / Sd - (W / Sd) ** 2, torch.ones_like(S0)).clamp_min(1e-300)
            ent = S * 0.5 * torch.log(two_pi * np.e * var1) + (1 - S) * 0.5 * torch.log(two_pi * np.e / Ea[None, :])
            total += float((lp + ent).sum())
            if ss:
                lnth, ln1mth = _E_beta(v.theta)
                S1 = (1 - S0).clamp(1e-300, 1.0)
                total += float((S0 * lnth[None, :] + (1 - S0) * ln1mth[None, :] - S0 * torch.log(S)
                                - (1 - S0) * torch.log(S1)).sum())
                total += _kl_beta(v.theta, TH_A0, TH_B0)
            if ard_w:
                total += _kl_gamma(v.alpha, A0, B0)
        if ard_f:
            Ea, Elna = _E_gamma(self.alphaZ)
        else:
            Ea, Elna = (torch.ones((G, K), dtype=f64, device=self.dev), torch.zeros((G, K), dtype=f64, device=self.dev))
        total += float((0.5 * self.Ng[:, None] * Elna - 0.5 * Ea * self.Ez2 + 0.5 * self.Ng[:, None]).sum())
        total += float((0.5 * self.class_count[:, None] * torch.log(self.zvar)).sum())
        if ard_f:
            total += _kl_gamma(self.alphaZ, A0, B0)
        return total

    def variance_explained(self):
        """R^2 (%) per view, group and factor from sufficient statistics: 1 - SS(Y - z_k w_k^T)/SS(Y)."""
        K = self.K
        out = []
        for v in self.views:
            W = v.W[:, :K].to(f64)
            r2 = torch.zeros((self.G, K), dtype=f64, device=self.dev)
            for g in range(self.G):
                P = v.P[g][:, :K].to(f64)
                if v.mu32 is not None:
                    P = P - v.mu64[g][:, None] * v.zsum[g][None, :]
                P = P * v.inv_scale[g]
                ss = v.ssq[g].sum()
                res = ss - 2.0 * (W * P).sum(0) + (W * W).sum(0) * torch.diagonal(v.ZZ_mean[g])
                r2[g] = 100.0 * (1.0 - res / ss) if float(ss) > 0 else 0.0
            out.append(r2)
        return out


def _train(model, n_iterations, convergence_mode, check_convergence, sort_factors, verbose):
    tol = TOLERANCE[convergence_mode]
    converged, it = False, -1
    for it in range(n_iterations):
        model.step()
        if verbose and _dist.rank() == 0:
            print(f"[mofa] iteration {it + 1}: ELBO = {model.elbo[-1]:.6e}")
        if check_convergence and it >= 1:
            delta = 100.0 * abs((model.elbo[-1] - model.elbo[-2]) / model.elbo[0])
            if delta < tol:
                converged = True
                break
    var = model.variance_explained()                       # list over views of G x K
    K = model.K
    order = torch.arange(K, device=model.dev)
    if sort_factors:
        order = torch.argsort(-torch.stack([x.sum(0) for x in var]).sum(0), stable=True)
    return {"Z": model.Z[:, :K][:, order], "W": [v.W[:, :K][:, order] for v in model.views],
            "variance": [x[:, order] for x in var], "elbo": model.elbo, "iterations": it + 1,
            "converged": converged, "order": order, "intercepts": [v.mean for v in model.views], "model": model}


def run_mofa_device(views, n_factors, n_iterations, n_total, Z0, center=True, scale_views=False, ard_weights=True,
                    ard_factors=True, spikeslab_weights=True, convergence_mode="fast", check_convergence=True,
                    sort_factors=True, verbose=False, likelihoods=None):
    """One group, every cell observed in every view (the benchmark case).  ``views``: per modality a DeviceCSR
    (gaussian) or a dense fp32 device tensor (poisson / bernoulli, see ``likelihoods``) of this rank's cells.
    Returns dict(Z, W (list), variance (list of K-vectors), elbo, iterations, converged)."""
    n_local = views[0].shape[0]
    blocks = [[(A, (0, n_local))] for A in views]
    model = MofaDevice(blocks, [A.shape[1] for A in views], [(0, n_local)], [n_total], None, n_factors, Z0, center,
                       scale_views, False, ard_weights, ard_factors, spikeslab_weights, likelihoods)
    res = _train(model, n_iterations, convergence_mode, check_convergence, sort_factors, verbose)
    res["variance"] = [x[0] for x in res["variance"]]
    res["intercepts"] = [x[0] for x in res["intercepts"]]
    return res


# ------------------------------------------------------------------------------------------------------
def _to_device_view(X):
    import scipy.sparse as sp
    if isinstance(X, _device.DeviceCSR):
        return X if X.data.dtype == torch.float32 else X.with_data(X.data.to(torch.float32))
    Xs = X.tocsr() if sp.issparse(X) else sp.csr_matrix(np.asarray(X))
    return _device.DeviceCSR.from_scipy(Xs, dtype=np.float32)


def _guess_likelihood(X) -> str:
    """mofapy2's ``guess_likelihoods`` (reached from muon/_core/tools.py:272-280) on one view: bernoulli if every
    value is 0 or 1, poisson if every value is an integer, else gaussian.  Implicit zeros of a sparse matrix are
    integers, so only the stored values need looking at (all of them, not a sample)."""
    if isinstance(X, _device.DeviceCSR):
        vals = X.data
        if vals.numel() == 0:
            return "bernoulli"
        if not bool((vals == vals.round()).all()):
            return "gaussian"
        return "bernoulli" if bool(((vals == 0) | (vals == 1)).all()) else "poisson"
    vals = X.data if hasattr(X, "data") and not isinstance(X, np.ndarray) else np.asarray(X).ravel()
    vals = np.asarray(vals)
    vals = vals[~np.isnan(vals)] if vals.dtype.kind == "f" else vals
    if vals.size and not np.all(vals == np.round(vals)):
        return "gaussian"
    return "bernoulli" if np.all((vals == 0) | (vals == 1)) else "poisson"


def _check_dense_fits(name, shape, lik, dev):
    """Non-gaussian views need dense N x D pseudo-data (observations + pseudo-data + zeta: 12 B per element)."""
    need = 12.0 * shape[0] * shape[1]
    free = torch.cuda.mem_get_info(dev)[0]
    if need > 0.6 * free:
        raise NotImplementedError(
            f"view '{name}' ({shape[0]} x {shape[1]}) was given / guessed the {lik} likelihood, whose pseudo-data are dense by "
            f"construction: {need / 2**30:.0f} GiB needed, {free / 2**30:.0f} GiB free on the device (the reference densifies "
            "every view and cannot run this size either).  Pass likelihoods='gaussian' for normalised data, or subset.")


def _to_dense_device(X, dev) -> torch.Tensor:
    """Any matrix -> dense row-major fp32 tensor on the device (the observations of a non-gaussian view)."""
    import scipy.sparse as sp
    if isinstance(X, torch.Tensor):
        return X.to(dev, torch.float32).contiguous()
    if isinstance(X, _device.DeviceCSR):
        t = torch.sparse_csr_tensor(X.indptr, X.indices.to(torch.int64), X.data.to(torch.float32), size=X.shape, device=dev)
        return t.to_dense().contiguous()
    arr = X.toarray() if sp.issparse(X) else np.asarray(X)
    if np.isnan(arr).any():
        raise NotImplementedError("missing values (NaN) inside a non-gaussian view are not supported; drop the cells "
                                  "from the view and use use_obs='union'")
    return torch.from_numpy(np.ascontiguousarray(arr, dtype=np.float32)).to(dev)


def mofa(
    data,
    groups_label=None,
    use_raw: bool = False,
    use_layer: Optional[str] = None,
    use_var: Optional[str] = "highly_variable",
    use_obs: Optional[str] = None,
    likelihoods=None,
    n_factors: int = 10,
    scale_views: bool = False,
    scale_groups: bool = False,
    center_groups: bool = True,
    ard_weights: bool = True,
    ard_factors: bool = True,
    spikeslab_weights: bool = True,
    spikeslab_factors: bool = False,
    n_iterations: int = 1000,
    convergence_mode: str = "fast",
    use_float32: bool = False,
    gpu_mode: bool = False,
    gpu_device=None,
    svi_mode: bool = False,
    svi_batch_size: float = 0.5,
    svi_learning_rate: float = 1.0,
    svi_forgetting_rate: float = 0.5,
    svi_start_stochastic: int = 1,
    smooth_covariate: Optional[str] = None,
    smooth_warping: bool = False,
    smooth_kwargs=None,
    save_parameters: bool = False,
    save_data: bool = True,
    save_metadata: bool = True,
    seed: int = 1,
    outfile: Optional[str] = None,
    expectations=None,
    save_interrupted: bool = True,
    verbose: bool = False,
    quiet: bool = True,
    copy: bool = False,
):
    """Run Multi-Omics Factor Analysis -- drop-in for ``muon.tl.mofa`` (muon/_core/tools.py:290-708).

    Writes ``obsm["X_mofa"]`` (cells x factors), ``varm["LFs"]`` (features x factors, zero rows for
    features excluded by ``use_var``), ``uns["mofa"]["params"]`` and ``uns["mofa"]["variance"]``
    ({view: R^2 per factor in %}), factors ordered by total variance explained.  Returns a copy when
    ``copy=True``, else ``None``.  ``gpu_mode``/``gpu_device`` are accepted and ignored (always GPU).
    """
    if is_anndata(data):
        mdata = SimpleMuData({"data": data})            # tools.py:425-431
        mdata.obs = data.obs
    elif is_mudata(data):
        mdata = data
    else:
        raise TypeError("Expected an MuData object")

    if use_var and (not hasattr(data.var, "columns") or use_var not in data.var.columns):
        # mudata lifts a .var column shared by every modality into mdata.var on update(); the test double does not,
        # so look at the modalities before concluding that the column is absent (tools.py:438-440)
        in_all_mods = is_mudata(data) and all(hasattr(a.var, "columns") and use_var in a.var.columns for a in mdata.mod.values())
        if not in_all_mods:
            warn(f"There is no column {use_var} in the provided object")
            use_var = None
    common_obs = None
    if is_mudata(data):
        common_obs = reduce(np.intersect1d, [np.asarray(v.obs_names) for v in mdata.mod.values()])
        if len(common_obs) != mdata.n_obs:
            if not use_obs:
                raise IndexError(
                    "Not all the observations are the same across modalities. Please run `mdata.intersect_obs()` "
                    "to subset the data or devise a strategy with `use_obs` ('union' or 'intersection')")
            elif use_obs not in ["union", "intersection"]:
                raise ValueError(f"Expected `use_obs` argument to be 'union' or 'intersection', not '{use_obs}'")
        else:
            use_obs = None

    for flag, name in ((svi_mode, "svi_mode"), (smooth_covariate, "smooth_covariate"),
                       (spikeslab_factors, "spikeslab_factors"), (use_raw, "use_raw")):
        if flag:
            raise NotImplementedError(f"mofa(..., {name}=...) is not supported by the CUDA path yet")
    lik = likelihoods
    if lik is not None:
        lik = [lik] * len(mdata.mod) if isinstance(lik, str) else list(lik)
        if len(lik) != len(mdata.mod) or any(l not in ("gaussian", "poisson", "bernoulli") for l in lik):
            raise ValueError(f"likelihoods must be 'gaussian', 'poisson' or 'bernoulli' per modality, got {likelihoods!r}")
    if groups_label is not None and (not hasattr(mdata.obs, "columns") or groups_label not in mdata.obs.columns):
        raise KeyError(f"{groups_label} is not in observations names")     # reference prints and exits, tools.py:98-101

    _device.require_cuda()
    import scipy.sparse as sp
    dev = torch.device("cuda", torch.cuda.current_device())
    mods = list(mdata.mod.keys())
    M = len(mods)
    obs_all = np.asarray(mdata.obs_names).astype(str)
    simple = (use_obs is None and groups_label is None and not scale_groups)

    # ---- features (tools.py:172-176) -----------------------------------------------------------------------
    Xs, masks = [], []
    for m in mods:
        adata = mdata.mod[m]
        X = adata.layers[use_layer] if use_layer else adata.X
        mask = None
        if use_var and hasattr(adata.var, "columns") and use_var in adata.var.columns:
            mask = np.asarray(adata.var[use_var].astype(bool))
            if isinstance(X, _device.DeviceCSR):
                raise NotImplementedError("use_var with a device-resident matrix is not supported yet")
            X = (X.tocsr() if sp.issparse(X) else np.asarray(X))[:, mask]
        elif use_var:
            mask = np.ones(adata.n_vars, dtype=bool)
        Xs.append(X)
        masks.append(mask)

    if lik is None:
        # The reference lets mofapy2 guess the likelihood per view (tools.py:272-280, mofapy2 guess_likelihoods):
        # all values in {0,1} -> bernoulli, all integers -> poisson, else gaussian.
        lik = [_guess_likelihood(X) for X in Xs]
    for m, X, l in zip(mods, Xs, lik):
        if l != "gaussian":
            _check_dense_fits(m, X.shape, l, dev)

    if simple:
        views = [_to_device_view(X) if l == "gaussian" else _to_dense_device(X, dev) for X, l in zip(Xs, lik)]
        sparse_views = [v for v in views if isinstance(v, _device.DeviceCSR)]
        n_local = views[0].shape[0]
        if sparse_views:
            n_total, row0 = sparse_views[0].n_total, sparse_views[0].row0
        elif _dist.is_distributed():
            raise NotImplementedError("cell-sharded mofa() needs at least one gaussian (DeviceCSR) view to carry the shard offsets")
        else:
            n_total, row0 = n_local, 0
        rs = np.random.RandomState(seed)
        Z0 = torch.from_numpy(rs.normal(size=(n_total, n_factors))[row0:row0 + n_local])
        res = run_mofa_device(views, n_factors, n_iterations, n_total, Z0, center=center_groups,
                              scale_views=scale_views, ard_weights=ard_weights, ard_factors=ard_factors,
                              spikeslab_weights=spikeslab_weights, convergence_mode=convergence_mode,
                              verbose=verbose and not quiet, likelihoods=lik)
        Z_full = res["Z"].cpu().numpy()
        group_names = ["group1"]
        variance = {m: res["variance"][i].cpu().numpy() for i, m in enumerate(mods)}
    else:
        # ---- general path: groups of cells and/or cells missing from whole views (host matrices) ---------------
        if any(isinstance(X, _device.DeviceCSR) for X in Xs) or _dist.is_distributed():
            raise NotImplementedError("groups_label / use_obs need host matrices on a single process for now")
        sel = obs_all if use_obs != "intersection" else obs_all[np.isin(obs_all, common_obs.astype(str))]
        if groups_label is not None:                       # groups in order of first appearance, tools.py:215-219
            glab_all = np.asarray(mdata.obs[groups_label]).astype(str)
            glab = glab_all[np.isin(obs_all, sel)] if len(sel) != len(obs_all) else glab_all
            group_names = list(dict.fromkeys(glab.tolist()))
        else:
            glab = np.array(["group1"] * len(sel))
            group_names = ["group1"]
        gid = np.array([group_names.index(x) for x in glab])
        perm = np.argsort(gid, kind="stable")               # cells ordered by group (tools.py:243-255)
        cells = sel[perm]
        gid = gid[perm]
        N = len(cells)
        G = len(group_names)
        bounds = np.searchsorted(gid, np.arange(G + 1))
        group_ranges = [(int(bounds[g]), int(bounds[g + 1])) for g in range(G)]
        pos_of = {c: i for i, c in enumerate(cells)}
        bits = np.zeros(N, dtype=np.int64)
        blocks, dims = [], []
        for mi, m in enumerate(mods):
            names = np.asarray(mdata.mod[m].obs_names).astype(str)
            X = Xs[mi]
            X = X.tocsr() if sp.issparse(X) else sp.csr_matrix(np.asarray(X))
            here = np.array([pos_of.get(c, -1) for c in names])     # position of each of the view's rows in Z
            keep = np.nonzero(here >= 0)[0]
            order = keep[np.argsort(here[keep], kind="stable")]      # view rows in Z order
            zpos = here[order]
            bits[zpos] |= (1 << mi)
            per_g = []
            for g, (lo, hi) in enumerate(group_ranges):
                selg = (zpos >= lo) & (zpos < hi)
                rows_z = zpos[selg]
                Xg = X[order[selg]].astype(np.float32)
                if lik[mi] == "gaussian":
                    A = _device.DeviceCSR.from_scipy(sp.csr_matrix(Xg), dtype=np.float32)
                else:
                    A = _to_dense_device(Xg, dev)
                if len(rows_z) == hi - lo and np.array_equal(rows_z, np.arange(lo, hi)):
                    per_g.append((A, (lo, hi)))
                else:
                    per_g.append((A, torch.from_numpy(rows_z.astype(np.int64)).to(dev)))
            blocks.append(per_g)
            dims.append(X.shape[1])
        cls = torch.from_numpy(((gid << M) | bits).astype(np.int32)).to(dev)
        rs = np.random.RandomState(seed)
        Z0 = torch.from_numpy(rs.normal(size=(N, n_factors)))
        model = MofaDevice(blocks, dims, group_ranges, [hi - lo for lo, hi in group_ranges], cls, n_factors, Z0,
                           center_groups, scale_views, scale_groups, ard_weights, ard_factors, spikeslab_weights, lik)
        res = _train(model, n_iterations, convergence_mode, True, True, verbose and not quiet)
        Zp = res["Z"].cpu().numpy()
        where = {c: i for i, c in enumerate(obs_all)}
        Z_full = np.full((len(obs_all), n_factors), np.nan)          # tools.py:617-622
        Z_full[[where[c] for c in cells]] = Zp
        if G > 1:                                                    # tools.py:690-697
            variance = {m: {group_names[g]: res["variance"][i][g].cpu().numpy() for g in range(G)}
                        for i, m in enumerate(mods)}
        else:
            variance = {m: res["variance"][i][0].cpu().numpy() for i, m in enumerate(mods)}

    if copy:
        data = data.copy()
    out_dt = np.float32 if use_float32 else np.float64
    data.obsm["X_mofa"] = Z_full.astype(out_dt)                                         # tools.py:616-628
    w = np.concatenate([W.cpu().numpy() for W in res["W"]], axis=0).astype(out_dt)
    if use_var:                                                                      # tools.py:636-641
        full = np.zeros((data.n_vars, w.shape[1]), dtype=out_dt)
        full[np.concatenate(masks)] = w
        data.varm["LFs"] = full
    else:
        data.varm["LFs"] = w
    data.uns["mofa"] = {
        "params": {
            "data": {"groups_label": groups_label, "use_raw": use_raw, "use_layer": use_layer,
                     "likelihoods": np.array(lik), "features_subset": use_var,
                     "use_obs": use_obs, "scale_views": scale_views, "scale_groups": scale_groups,
                     "center_groups": center_groups, "use_float32": use_float32},
            "model": {"ard_factors": ard_factors, "ard_weights": ard_weights, "spikeslab_weights": spikeslab_weights,
                      "spikeslab_factors": spikeslab_factors, "n_factors": n_factors},
            "training": {"n_iterations": n_iterations, "convergence_mode": convergence_mode, "gpu_mode": gpu_mode,
                         "seed": seed},
        },
        "variance": variance,
    }
    data.uns["mofa"]["_b200"] = {"iterations": res["iterations"], "converged": res["converged"], "elbo": res["elbo"]}
    if copy:
        return data
    if not quiet:
        print("Saved MOFA embeddings in .obsm['X_mofa'] slot and their loadings in .varm['LFs'].")
    return None
