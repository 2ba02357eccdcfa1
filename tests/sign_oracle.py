"""FP64 spec of dfm_sign_restrictions: shocks identified by sign restrictions on the series responses of a state-space DFM.
ORACLE / TEST INFRASTRUCTURE ONLY (NumPy; checked in tests/test_oracle_sign.py).

One model (Lam N x r, R N, A r x k, Q r x r): L = chol(Q), Psi_h = [M^h]_{1:r,1:r} L (identified_oracle.psi), c_{i,h} = lam_i' Psi_h.
  Rows (i, h, j, s): series i, horizon h, shock j (1-based), sign s = +1 / -1.
  Candidate c of model id: Z[a, j] = rng_normal(seed, id, 18, c r^2 + a + r j); Z = Q_Z R_Z (numpy.linalg.qr),
  Omega = Q_Z diag(sign(diag R_Z)).
  Acceptance: for each shock j with rows, v = s c_{i,h} omega_j over its rows: all > 0 keep, all < 0 flip omega_j, else reject.
  The first n_keep accepted candidates (candidate order) are kept: cand, rot = Omega (flips applied),
  resp[i,h,j] = scale_i c_{i,h} Omega e_j, fevd[i,h,j] = sum_{l<=h} (c_{i,l} Omega e_j)^2 / (sum_{l<=h} |c_{i,l}|^2 + R_i).
  Status 3: A or Q holds a NaN or Q is not positive definite; 1: a restricted series is out of the model.  Such a model accepts
  nothing.  Empty slots: cand -1, NaN rot / resp / fevd.
"""
import numpy as np

import identified_oracle as IO
from gibbs_oracle import in_model
from oracle.dgp import rng_normal

RNG_SIGN = 18


def omegas(seed, mid, c, r):
    """Omega of candidates c (array) of model id `mid`: (len(c), r, r)."""
    c = np.asarray(c, dtype=np.uint64).reshape(-1)
    e = c[:, None] * np.uint64(r * r) + np.arange(r * r, dtype=np.uint64)[None, :]
    Z = rng_normal(seed, mid, RNG_SIGN, e.ravel()).reshape(len(c), r, r).transpose(0, 2, 1)     # Z[c, a, j], element a + r j
    Qz, Rz = np.linalg.qr(Z)
    return Qz * np.sign(np.diagonal(Rz, axis1=1, axis2=2))[:, None, :]


def row_vectors(Lam, A, Q, p, rows, H):
    """s c_{i,h} of every row, (n, r)."""
    P = IO.psi(A, Q, p, H)
    return np.array([s * (np.asarray(Lam, float)[i] @ P[h]) for i, h, j, s in rows]).reshape(len(rows), Lam.shape[1])


def decide(C, shocks, Om):
    """Per candidate: accepted (n_cand,), the flips (n_cand, r) and the smallest |v| / |c| over the rows of the shocks each
    candidate reaches (its first failing shock included)."""
    nc, r = Om.shape[0], Om.shape[1]
    ok = np.ones(nc, bool); flip = np.ones((nc, r)); margin = np.full(nc, np.inf)
    for j in sorted(set(shocks)):
        sel = np.flatnonzero(np.asarray(shocks) == j)
        v = np.einsum("qa,ca->cq", C[sel], Om[:, :, j - 1])
        rel = np.min(np.abs(v) / np.linalg.norm(C[sel], axis=1)[None, :], axis=1)
        margin = np.where(ok, np.minimum(margin, rel), margin)
        pos, neg = (v > 0).all(1), (v < 0).all(1)
        flip[:, j - 1] = np.where(neg, -1.0, 1.0)
        ok &= pos | neg
    return ok, flip, margin


def identify(Lam, R, A, Q, p, rows, H, n_shock, n_rot, n_keep, seed=0, mid=0, scale=None):
    """dfm_sign_restrictions on one model: dict n_accept, cand (n_keep,), rot (n_keep, r, r), resp / fevd (n_keep, N, H, n_shock),
    status, and margin (the smallest relative |v| over every row a candidate tests)."""
    Lam = np.asarray(Lam, float); R = np.asarray(R, float); N, r = Lam.shape
    out = dict(n_accept=0, cand=np.full(n_keep, -1), rot=np.full((n_keep, r, r), np.nan), resp=np.full((n_keep, N, H, n_shock), np.nan),
               fevd=np.full((n_keep, N, H, n_shock), np.nan), status=0, margin=np.inf)
    if np.isnan(A).any() or np.isnan(Q).any():
        out["status"] = 3
        return out
    try:
        P = IO.psi(A, Q, p, H)
    except np.linalg.LinAlgError:
        out["status"] = 3
        return out
    inm = in_model(Lam, R)
    if any(not inm[i] for i, h, j, s in rows):
        out["status"] = 1
        return out
    C = row_vectors(Lam, A, Q, p, rows, H)
    shocks = [j for i, h, j, s in rows]
    Om = omegas(seed, mid, np.arange(n_rot), r)
    ok, flip, margin = decide(C, shocks, Om)
    out["margin"] = float(margin.min()) if len(margin) else np.inf
    acc = np.flatnonzero(ok)
    out["n_accept"] = len(acc)
    kept = acc[:n_keep]
    out["cand"][:len(kept)] = kept
    Omk = Om[kept] * flip[kept][:, None, :]
    out["rot"][:len(kept)] = Omk
    if len(kept):
        out["resp"][:len(kept)], out["fevd"][:len(kept)] = rotated_responses(Lam, R, P, Omk, n_shock, scale)
    return out


def rotated_responses(Lam, R, P, Om, n_shock, scale=None):
    """resp, fevd (n, N, H, n_shock) of the rotations Om (n, r, r) at Psi P (H, r, r)."""
    Lam = np.asarray(Lam, float); R = np.asarray(R, float); N = Lam.shape[0]
    c = np.einsum("ia,hab->ihb", Lam, P)                                        # (N, H, r)
    den = np.cumsum(c ** 2, axis=1).sum(axis=2) + R[:, None]
    sc = np.ones(N) if scale is None else np.asarray(scale, float)
    cr = np.einsum("ihb,nbj->nihj", c, Om[:, :, :n_shock])
    resp = sc[None, :, None, None] * cr
    fevd = np.cumsum(cr ** 2, axis=2) / den[None, :, :, None]
    out = ~in_model(Lam, R)
    resp[:, out] = np.nan; fevd[:, out] = np.nan
    return resp, fevd


def acceptance(C, shocks, seed, mid, n_rot):
    """Share of the first n_rot candidates accepted (r from C)."""
    Om = omegas(seed, mid, np.arange(n_rot), C.shape[1])
    return decide(C, shocks, Om)[0].mean()
