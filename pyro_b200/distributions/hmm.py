"""GaussianHMM (SURVEY.md row c1, BASELINE config 3).

Interface mirrors pyro/distributions/hmm.py:434-582 (constructor arguments, shapes, ``log_prob``).
The reference eliminates the time axis with a parallel scan of Gaussian tensordots
(pyro/ops/gaussian.py:510-597): O(log T) depth but O(T (2H)^3) work and a materialised
``[T, 2H, 2H]`` precision tensor (41.9 GB at H=512, T=10 000).  Here ``log_prob`` is the
mathematically identical marginal likelihood computed by the innovation form of the Kalman
filter: O(T H^3) work, O(H^2) live state, and every heavy operation is a dense ``H x H`` GEMM.

Round-1 status: the GEMMs / small Choleskys run through cuBLAS / cuSOLVER (``torch.matmul``,
``torch.linalg``) -- plain library contractions, fp32 (or TF32 tensor cores with ``tf32=True``) --
and gradients come from autograd through the recursion.  There is no hand-written tensor-core kernel
for this row yet (DESIGN.md section 7); parity with the reference is pinned by
tests/golden/hmm.npz.
"""
import math

import torch
from torch.distributions import constraints

from . import Distribution, Independent, MultivariateNormal, Normal


def _loc_cov(d):
    """(loc, covariance) of a MultivariateNormal or an Independent(Normal, 1)."""
    if isinstance(d, MultivariateNormal):
        L = d.scale_tril
        return d.loc, L @ L.transpose(-1, -2)
    if isinstance(d, Independent) and isinstance(d.base_dist, Normal) and d.reinterpreted_batch_ndims == 1:
        base = d.base_dist
        shape = base.batch_shape
        loc = base.loc.expand(shape)
        var = (base.scale ** 2).expand(shape)
        return loc, torch.diag_embed(var)
    if hasattr(d, "loc") and hasattr(d, "covariance_matrix"):  # a torch.distributions MVN
        return d.loc, d.covariance_matrix
    raise ValueError("expected a MultivariateNormal or Normal(...).to_event(1), got {}".format(type(d).__name__))


class GaussianHMM(Distribution):
    has_rsample = True
    arg_constraints = {}
    support = constraints.independent(constraints.real, 2)

    def __init__(self, initial_dist, transition_matrix, transition_dist, observation_matrix,
                 observation_dist, validate_args=None, duration=None, tf32=False, steady_state=True):
        hidden_dim, obs_dim = observation_matrix.shape[-2:]
        self.hidden_dim, self.obs_dim = hidden_dim, obs_dim
        self.duration = duration
        self.tf32 = tf32
        self.steady_state = steady_state   # time-invariant parameters: blocked scan after the covariance converges
        self._m0, self._P0 = _loc_cov(initial_dist)
        self._F = transition_matrix
        self._bw, self._Q = _loc_cov(transition_dist)
        self._H = observation_matrix
        self._bv, self._R = _loc_cov(observation_dist)
        assert self._m0.shape[-1] == hidden_dim and self._F.shape[-2:] == (hidden_dim, hidden_dim)
        assert self._bw.shape[-1] == hidden_dim and self._bv.shape[-1] == obs_dim
        shape = torch.broadcast_shapes(self._m0.shape[:-1] + (1,), self._F.shape[:-2], self._bw.shape[:-1],
                                       self._H.shape[:-2], self._bv.shape[:-1])
        batch_shape, time_shape = shape[:-1], shape[-1:]
        if duration is not None and time_shape[0] == 1:
            time_shape = torch.Size((duration,))
        super().__init__(batch_shape, time_shape + (obs_dim,))

    def expand(self, batch_shape, _instance=None):
        new = GaussianHMM.__new__(GaussianHMM)
        new.__dict__.update(self.__dict__)
        new._batch_shape = torch.Size(torch.broadcast_shapes(self.batch_shape, torch.Size(batch_shape)))
        return new

    # time-dependent parameters carry the time axis at dim -3 (matrices) / -2 (vectors)
    @staticmethod
    def _at(x, t, mat):
        tdim = -3 if mat else -2
        if x.dim() >= -tdim and x.shape[tdim] != 1:
            return x.select(tdim, t)
        if x.dim() >= -tdim:
            return x.squeeze(tdim)
        return x

    def log_prob(self, value):
        T = value.shape[-2]
        # The GEMMs follow the AMBIENT ``torch.backends.cuda.matmul.allow_tf32`` setting in both the
        # forward and the autograd backward pass (default: fp32).  No global flag is touched here: a
        # forward-only toggle would leave the backward at a different precision and is not thread-safe
        # (ADVICE r1).  ``tf32=True`` is honoured only by asserting that the caller enabled it.
        if self.tf32 and not torch.backends.cuda.matmul.allow_tf32:
            raise ValueError("GaussianHMM(tf32=True): enable torch.backends.cuda.matmul.allow_tf32 around the "
                             "whole forward AND backward pass yourself")
        if self.steady_state and T >= 64 and value.dim() == 2 and self._homogeneous():
            return self._filter_steady(value, T)
        return self._filter(value, T)

    def _homogeneous(self):
        """Time-invariant, unbatched parameters (BASELINE config 3): the covariance recursion does not
        see the data and converges to the stationary Riccati solution."""
        return (len(self.batch_shape) == 0 and self._m0.dim() == 1 and self._P0.dim() == 2
                and self._F.dim() == 2 and self._H.dim() == 2 and self._bw.dim() == 1 and self._bv.dim() == 1
                and self._Q.dim() == 2 and self._R.dim() == 2)

    def _filter_steady(self, value, T):
        """Same marginal likelihood for time-invariant parameters in two phases.

        Phase 1 runs the exact recursion of ``_filter`` until the predicted covariance stops changing
        (relative max-norm change <= 1e-13 in fp64, 3e-7 in fp32 -- below the rounding of the sum it
        feeds).  From there the gain K, the innovation covariance S and the closed-loop matrix
        ``A = (I - H K) F`` are constants, so the predicted means obey the LINEAR recurrence
        ``m_{t+1} = m_t A + u_t`` with ``u_t = (x_t - b_v) K F + b_w``: phase 2 evaluates it as a
        blocked scan -- B dense steps shared by all blocks, a carry over the block starts with A^B, and
        one batched product with the stored powers -- i.e. O(sqrt(T)) sequential GEMMs instead of T
        steps of ~20 small kernels.  The H^3 FLOPs of the skipped covariance steps are NOT performed
        (SURVEY.md 8d: report them as skipped, not as achieved)."""
        F, Hm, bw, bv, Q, R = self._F, self._H, self._bw, self._bv, self._Q, self._R
        O, Hd = self.obs_dim, self.hidden_dim
        const = O * math.log(2 * math.pi)
        tol = 1e-13 if value.dtype == torch.float64 else 3e-7
        m = self._m0.unsqueeze(0)             # [1, H] predicted/filtered mean (row vector)
        P = self._P0
        Ft, Ht = F.transpose(-1, -2), Hm.transpose(-1, -2)
        Pm_prev = None
        t = 0
        converged = False
        vs_all, diag_all = [], []
        # The step is launch-bound (H = 512: ~20 small kernels per time step, three times that with the backward
        # pass), so the recursion is written with fused multiply-adds (addmm), the per-step likelihood terms are
        # only COLLECTED here and reduced once after the loop, and convergence is tested every 4th step (a test
        # is 6 launches and a host synchronisation; running up to 3 exact steps more costs less).
        while t < T:
            m = torch.addmm(bw, m, F)
            Pm = torch.addmm(Q, Ft @ P, F)
            if Pm_prev is not None and t >= 4 and t % 4 == 0:
                with torch.no_grad():
                    rel = float((Pm - Pm_prev).abs().max() / Pm.abs().max().clamp(min=1e-300))
                if rel <= tol:
                    converged = True
                    break
            PH = Pm @ Hm
            S = torch.addmm(R, Ht, PH)
            v = value[t:t + 1, :] - torch.addmm(bv, m, Hm)
            Ls = torch.linalg.cholesky(S)
            vs_all.append(torch.linalg.solve_triangular(Ls, v.transpose(-1, -2), upper=False))
            diag_all.append(Ls.diagonal())
            Kt = torch.cholesky_solve(PH.transpose(-1, -2), Ls)
            m = torch.addmm(m, v, Kt)
            P = torch.addmm(Pm, PH, Kt, alpha=-1.0)
            P = 0.5 * (P + P.transpose(-1, -2))
            Pm_prev = Pm
            t += 1
        ll = value.new_zeros(())
        if vs_all:
            VS = torch.cat(vs_all, dim=1)                                  # [O, t]
            ll = -0.5 * ((VS * VS).sum() + len(vs_all) * const) - torch.stack(diag_all).log().sum()
        if not converged:
            return ll
        # ---- stationary phase: m holds the predicted mean of step t, Pm the stationary covariance ----
        rem = T - t
        PH = Pm @ Hm
        S = torch.addmm(R, Ht, PH)
        Ls = torch.linalg.cholesky(S)
        Kt = torch.cholesky_solve(PH.transpose(-1, -2), Ls)            # [O, H]
        KF = Kt @ F                                                    # [O, H]
        A = F - Hm @ KF                                                # (I - H K) F
        X = value[t:] - bv                                             # [rem, O]
        U = torch.addmm(bw, X, KF)                                     # [rem, H]
        B = max(8, int(math.ceil(math.sqrt(rem))))
        nblk = (rem + B - 1) // B
        pad = nblk * B - rem
        if pad:
            U = torch.cat([U, U.new_zeros(pad, Hd)], dim=0)
        Ub = U.reshape(nblk, B, Hd)
        # powers A^1 .. A^B by doubling: [A^1..A^k] @ A^k = [A^(k+1)..A^(2k)] -- ceil(log2 B) batched GEMM launches
        # instead of B sequential ones (same FLOPs)
        pows = A.unsqueeze(0)
        while pows.shape[0] < B:
            k = pows.shape[0]
            take = min(k, B - k)
            pows = torch.cat([pows, pows[:take] @ pows[k - 1]], dim=0)
        AP = torch.cat([torch.eye(Hd, dtype=A.dtype, device=A.device).unsqueeze(0), pows[:B - 1]], dim=0)  # A^0..A^(B-1)
        AB = pows[B - 1]                                               # A^B
        # local solutions with zero start, all blocks at once
        w = U.new_zeros(nblk, Hd)
        Ws = []
        for j in range(B):
            Ws.append(w)
            w = torch.addmm(Ub[:, j], w, A)
        W = torch.stack(Ws, dim=1)                                     # [nblk, B, H]
        starts = []
        s_b = m                                                        # [1, H]
        for b in range(nblk):
            starts.append(s_b)
            s_b = torch.addmm(w[b:b + 1], s_b, AB)
        S0 = torch.cat(starts, dim=0)                                  # [nblk, H]
        M = torch.einsum("bh,jhk->bjk", S0, AP) + W                    # predicted means [nblk, B, H]
        M = M.reshape(nblk * B, Hd)[:rem]
        V = X - M @ Hm                                                 # innovations [rem, O]
        vs = torch.linalg.solve_triangular(Ls, V.transpose(-1, -2), upper=False)
        ll = ll - 0.5 * ((vs * vs).sum() + rem * const) - rem * Ls.diagonal().log().sum()
        return ll

    def filter(self, value):
        """Posterior over the FINAL hidden state given a sequence of observations, as a ``MultivariateNormal``
        usable as ``initial_dist`` of a continuation (pyro/distributions/hmm.py:604-633: there the time axis is
        eliminated by the tensordot scan and the precision form is converted back; here the filtered mean and
        covariance of the last Kalman step are the answer directly)."""
        T = value.shape[-2]
        _, m, P = self._filter(value, T, return_state=True)
        return MultivariateNormal(m.squeeze(-2), covariance_matrix=P)

    def _filter(self, value, T, return_state=False):
        O = self.obs_dim
        m = self._m0.unsqueeze(-2)            # [..., 1, H] row vector
        P = self._P0
        ll = 0.0
        const = O * math.log(2 * math.pi)
        for t in range(T):
            F = self._at(self._F, t, True)
            Hm = self._at(self._H, t, True)
            bw = self._at(self._bw, t, False).unsqueeze(-2)
            bv = self._at(self._bv, t, False).unsqueeze(-2)
            Q = self._at(self._Q, t, True)
            R = self._at(self._R, t, True)
            # predict:  z_t = z_{t-1} F + w
            m = m @ F + bw
            P = F.transpose(-1, -2) @ P @ F + Q
            # innovation:  x_t = z_t H + v
            PH = P @ Hm                                     # [..., H, O]
            S = Hm.transpose(-1, -2) @ PH + R               # [..., O, O]
            v = value[..., t:t + 1, :] - (m @ Hm + bv)      # [..., 1, O]
            Ls = torch.linalg.cholesky(S)
            vs = torch.linalg.solve_triangular(Ls, v.transpose(-1, -2), upper=False)   # [..., O, 1]
            ll = ll - 0.5 * ((vs * vs).sum((-1, -2)) + const) - Ls.diagonal(dim1=-2, dim2=-1).log().sum(-1)
            # update
            Kt = torch.cholesky_solve(PH.transpose(-1, -2), Ls)                        # S^-1 H^T P  [..., O, H]
            m = m + v @ Kt
            P = P - PH @ Kt
            P = 0.5 * (P + P.transpose(-1, -2))
        if return_state:
            return ll, m, P
        return ll

    def rsample(self, sample_shape=torch.Size()):
        T = self.event_shape[0] if self.duration is None else self.duration
        shape = torch.Size(sample_shape) + self.batch_shape
        L0 = torch.linalg.cholesky(self._P0)
        z = self._m0 + (L0 @ torch.randn(shape + (self.hidden_dim, 1), dtype=L0.dtype, device=L0.device)).squeeze(-1)
        xs = []
        for t in range(T):
            Lq = torch.linalg.cholesky(self._at(self._Q, t, True))
            Lr = torch.linalg.cholesky(self._at(self._R, t, True))
            w = (Lq @ torch.randn(shape + (self.hidden_dim, 1), dtype=L0.dtype, device=L0.device)).squeeze(-1)
            z = (z.unsqueeze(-2) @ self._at(self._F, t, True)).squeeze(-2) + self._at(self._bw, t, False) + w
            e = (Lr @ torch.randn(shape + (self.obs_dim, 1), dtype=L0.dtype, device=L0.device)).squeeze(-1)
            xs.append((z.unsqueeze(-2) @ self._at(self._H, t, True)).squeeze(-2) + self._at(self._bv, t, False) + e)
        return torch.stack(xs, dim=-2)
