"""The reprojection-outlier rule of lvba_visual_remove_outliers / lvba_visual_remove_observations, restated twice: a literal
per-landmark loop and a vectorised numpy form (include/lvba_b200.h, B2).

Observations are named by the caller's index q into obs_cam / obs_uv as given at create.  An observation is in the problem
while its landmark has a valid plane and has not been dropped, and it has not been removed.  At the current state, for every
observation in the problem, s_q = r0^2 + r1^2 (the term the cost sums before any loss):
  1. tau = (max_err_px / sigma_px)^2;
  2. an observation in the problem is removed iff !(z > 1e-8 and s_q <= tau): the cut-off case (s_q = +inf here), NaN and
     s_q > tau are removed, s_q == tau is kept;
  3. a landmark left with fewer than min_track_len observations in the problem is dropped: its remaining observations are
     removed too, its plane leaves the cost, and its X stays.
With a caller mask instead of step 2 (remove_observations), the flagged observations in the problem are removed; flags on
observations out of the problem are ignored."""
import numpy as np

from oracle import visual_oracle as vo


def obs_sq(q, t, X, obs_ptr, obs_cam, obs_uv, intr, sigma_px, in_problem):
    """s_q [N_obs] at (q, t, X): +inf where the depth fails z > 1e-8, NaN where in_problem [N_obs] is false"""
    obs_ptr = np.asarray(obs_ptr, np.int64)
    N = int(obs_ptr[-1])
    trk = np.repeat(np.arange(len(obs_ptr) - 1), np.diff(obs_ptr))
    cam = np.asarray(obs_cam, np.int64)
    uv = np.asarray(obs_uv, np.float32).astype(np.float64).reshape(N, 2)
    r, _, _, _ = vo.reproj_eval(q[cam], t[cam], X[trk], uv, intr, sigma_px, want_jac=False)
    z = (vo.quat_rotate(q[cam], X[trk]) + t[cam])[:, 2]
    s = r[:, 0] * r[:, 0] + r[:, 1] * r[:, 1]
    s = np.where(z > 1e-8, s, np.inf)
    return np.where(in_problem, s, np.nan)


def tau_of(max_err_px, sigma_px):
    e = max_err_px / sigma_px
    return min(e * e, np.finfo(np.float64).max)


def rule_loop(obs_ptr, in_problem, lm_in_problem, min_track_len, sq=None, tau=None, mask=None):
    """The literal loop: per landmark, its observations in the problem, the kept ones, the drop.  Returns (removed [N_obs],
    dropped [T]) of this call."""
    obs_ptr = np.asarray(obs_ptr, np.int64)
    T = len(obs_ptr) - 1
    removed = np.zeros(int(obs_ptr[-1]), bool)
    dropped = np.zeros(T, bool)
    for i in range(T):
        if not lm_in_problem[i]:
            continue
        here = [q for q in range(obs_ptr[i], obs_ptr[i + 1]) if in_problem[q]]
        if mask is None:
            kept = [q for q in here if sq[q] <= tau]           # NaN and +inf fail <=
        else:
            kept = [q for q in here if not mask[q]]
        if len(kept) < min_track_len:
            kept = []
            dropped[i] = True
        for q in here:
            if q not in kept:
                removed[q] = True
    return removed, dropped


def rule_vec(obs_ptr, in_problem, lm_in_problem, min_track_len, sq=None, tau=None, mask=None):
    """rule_loop in numpy"""
    obs_ptr = np.asarray(obs_ptr, np.int64)
    T = len(obs_ptr) - 1
    trk = np.repeat(np.arange(T), np.diff(obs_ptr))
    with np.errstate(invalid="ignore"):
        ok = (sq <= tau) if mask is None else ~np.asarray(mask, bool)
    keep = np.asarray(in_problem, bool) & ok
    cnt = np.bincount(trk[keep], minlength=T)
    dropped = np.asarray(lm_in_problem, bool) & (cnt < min_track_len)
    keep &= ~dropped[trk]
    return np.asarray(in_problem, bool) & ~keep, dropped


class Tracker:
    """What is in the problem after a sequence of removals: a caller's problem (dict with plane_nd, obs_ptr, obs_cam,
    obs_uv, ...) and the observations / landmarks taken out so far."""

    def __init__(self, p):
        self.p = p
        self.obs_ptr = np.asarray(p["obs_ptr"], np.int64)
        self.T = len(self.obs_ptr) - 1
        self.lm_in = vo.valid_tracks(np.asarray(p["plane_nd"], np.float64))
        trk = np.repeat(np.arange(self.T), np.diff(self.obs_ptr))
        self.obs_in = self.lm_in[trk].copy()

    def sq(self, q, t, X):
        p = self.p
        return obs_sq(q, t, X, p["obs_ptr"], p["obs_cam"], p["obs_uv"], p["intr"], p["sigma_px"], self.obs_in)

    def apply(self, removed, dropped):
        self.obs_in &= ~removed
        self.lm_in &= ~dropped

    def remove_outliers(self, q, t, X, max_err_px, min_track_len=3):
        sq = self.sq(q, t, X)
        rm, dr = rule_vec(self.obs_ptr, self.obs_in, self.lm_in, min_track_len, sq=sq, tau=tau_of(max_err_px, self.p["sigma_px"]))
        self.apply(rm, dr)
        return rm, dr

    def remove_observations(self, mask, min_track_len=3):
        rm, dr = rule_vec(self.obs_ptr, self.obs_in, self.lm_in, min_track_len, mask=mask)
        self.apply(rm, dr)
        return rm, dr

    def kept_problem(self):
        """The caller-compacted arrays a fresh lvba_visual_create would take for what is in the problem: the kept
        observations in the caller's order, every landmark out of the problem without a plane (n = 0, d = 0)."""
        p = dict(self.p)
        trk = np.repeat(np.arange(self.T), np.diff(self.obs_ptr))
        k = self.obs_in
        p["obs_ptr"] = np.concatenate([[0], np.cumsum(np.bincount(trk[k], minlength=self.T))]).astype(np.int64)
        p["obs_cam"] = np.ascontiguousarray(np.asarray(self.p["obs_cam"])[k], np.int32)
        p["obs_uv"] = np.ascontiguousarray(np.asarray(self.p["obs_uv"], np.float32).reshape(-1, 2)[k])
        pl = np.array(self.p["plane_nd"], np.float64)
        pl[~self.lm_in] = 0.0
        p["plane_nd"] = pl
        return p
