"""FP64 spec of dfm_narrative_sign_restrictions: sign restrictions plus narrative restrictions on dated episodes, with the
importance weight of every kept draw.  ORACLE / TEST INFRASTRUCTURE ONLY (NumPy; checked in tests/test_oracle_narrative.py).

One model (Lam N x r, R N, A r x k, Q r x r) and a factor path F (Tp x r): L = chol(Q), Psi_h (identified_oracle.psi, explicit
matrix powers), c_{i,h} = lam_i' Psi_h, u_t = L^-1 (f_t - sum_l A_l f_{t-l}) (t >= p).  Candidate Omega: sign_oracle's QR path.
  eps~_t = Omega' u_t;  H_{i,k}(t, h) = sum_{l=0..h} (c_{i,l} omega_k)(omega_k' u_{t+h-l})   (explicit convolution).
Narrative rows (kind, shock j 1-based, series i, row t, window h, sign s):
  0 s eps~_{j,t} > 0;  1 |H_j| > max_{k != j} |H_k|;  2 |H_j| > sum_{k != j} |H_k|;  3 s H_j > 0.
Acceptance per shock j: its sign rows fix the orientation (all > 0 keep, all < 0 flip), else its kind-0 rows do; kind-0 rows
are tested at that orientation, kind-3 rows as they are (H is quadratic in omega_j); kinds 1 / 2 on the whole Omega.
Weight: e_{k,tau} = rng_normal(seed, id, 19, (s nP + p) r + k), p the position of tau in the sorted union of the rows'
periods; n_ok = simulations that satisfy every row with H^sim_{i,k} = sum_l (c_{i,l} omega_k) e_{k,t+h-l}; weight n_sim / n_ok.
Weighted bands: per quantile the first sorted record whose exact cumulative weight reaches q / 100 of the total (Python
integers).
"""
import itertools

import numpy as np

import identified_oracle as IO
import sign_oracle as SO
from gibbs_oracle import in_model
from oracle.dgp import rng_normal

RNG_NARR = 19
KINDS = dict(shock=0, most=1, overwhelming=2, contrib=3)


def shocks_u(A, Q, F, p):
    """u_t (Tp, r), NaN for t < p."""
    F = np.asarray(F, float); Tp, r = F.shape
    L = np.linalg.cholesky(Q)
    U = np.full((Tp, r), np.nan)
    for t in range(p, Tp):
        v = F[t] - sum(A[:, (l - 1) * r:l * r] @ F[t - l] for l in range(1, p + 1))
        U[t] = np.linalg.solve(L, v)
    return U


def contributions(c, Om, U, t, h):
    """H_k (r,) of series with responses c (H, r) over rows t .. t+h, by explicit convolution."""
    r = Om.shape[1]
    return np.array([sum((c[l] @ Om[:, k]) * (Om[:, k] @ U[t + h - l]) for l in range(h + 1)) for k in range(r)])


def periods(narr):
    """The sorted union of the rows' periods and each row's position map."""
    ps = sorted({tau for kd, j, i, t, h, s in narr for tau in range(t, t + (0 if kd == 0 else h) + 1)})
    return ps, {tau: q for q, tau in enumerate(ps)}


def _share(kd, Hk, j):
    a = np.abs(Hk); o = np.delete(a, j)
    rhs = (o.max() if len(o) else 0.0) if kd == 1 else o.sum()
    return a[j] > rhs, abs(a[j] - rhs) / max(a.sum(), 1e-300)


def decide(Om, C, sign_shocks, narr, c_of, U, n_shock):
    """One candidate Omega (r, r): (accepted, flips (r,), smallest relative decision margin)."""
    r = Om.shape[0]
    flip = np.ones(r); margin = np.inf
    for j in range(1, n_shock + 1):
        w = Om[:, j - 1]
        f = 0
        sel = [q for q, sj in enumerate(sign_shocks) if sj == j]
        if sel:
            v = C[sel] @ w
            margin = min(margin, np.min(np.abs(v) / np.linalg.norm(C[sel], axis=1)))
            f = 1 if (v > 0).all() else (-1 if (v < 0).all() else 0)
            if f == 0:
                return False, flip, margin
        k0 = [row for row in narr if row[0] == 0 and row[1] == j]
        if k0:
            v = np.array([s * (U[t] @ w) for _, _, _, t, _, s in k0])
            margin = min(margin, np.min(np.abs(v) / np.array([np.linalg.norm(U[t]) for _, _, _, t, _, _ in k0])))
            g = 1 if (v > 0).all() else (-1 if (v < 0).all() else 0)
            if (f == 0 and g == 0) or (f != 0 and g != f):
                return False, flip, margin
            f = f or g
        flip[j - 1] = f or 1
        for kd, _, i, t, h, s in (row for row in narr if row[0] == 3 and row[1] == j):
            Hk = contributions(c_of(i), Om, U, t, h)
            margin = min(margin, abs(Hk[j - 1]) / max(np.abs(Hk).sum(), 1e-300))
            if not s * Hk[j - 1] > 0:
                return False, flip, margin
    for kd, j, i, t, h, s in (row for row in narr if row[0] in (1, 2)):
        ok, m = _share(kd, contributions(c_of(i), Om, U, t, h), j - 1)
        margin = min(margin, m)
        if not ok:
            return False, flip, margin
    return True, flip, margin


def decide_batch(Om, C, sign_shocks, narr, c_of, U, n_shock):
    """decide over candidates Om (n, r, r) at once: accepted (n,), flips (n, r), and each candidate's margin over the tests it
    reaches (its first failing test included), as decide's.  The contributions are the quadratic forms omega_k' G omega_k, G =
    sum_l c_l' u_{t+h-l}', in place of decide's explicit convolution."""
    n, r = Om.shape[0], Om.shape[1]
    ok = np.ones(n, bool); flip = np.ones((n, r)); margin = np.full(n, np.inf)

    def test(passed, m):
        nonlocal ok, margin
        margin = np.where(ok, np.minimum(margin, m), margin)
        ok = ok & passed

    def quad(i, t, h):                                          # H_k (n, r)
        c = c_of(i)
        G = sum(np.outer(c[l], U[t + h - l]) for l in range(h + 1))
        return np.einsum("nak,ab,nbk->nk", Om, G, Om)

    for j in range(1, n_shock + 1):
        w = Om[:, :, j - 1]
        f = np.zeros(n)
        sel = [q for q, sj in enumerate(sign_shocks) if sj == j]
        if sel:
            v = w @ C[sel].T
            pos, neg = (v > 0).all(1), (v < 0).all(1)
            test(pos | neg, np.min(np.abs(v) / np.linalg.norm(C[sel], axis=1), axis=1))
            f = np.where(pos, 1.0, np.where(neg, -1.0, 0.0))
        k0 = [row for row in narr if row[0] == 0 and row[1] == j]
        if k0:
            v = np.stack([s * (w @ U[t]) for _, _, _, t, _, s in k0], 1)
            g = np.where((v > 0).all(1), 1.0, np.where((v < 0).all(1), -1.0, 0.0))
            test(np.where(f == 0, g != 0, g == f), np.min(np.abs(v) / np.array([np.linalg.norm(U[t]) for _, _, _, t, _, _ in k0]), axis=1))
            f = np.where(f == 0, g, f)
        flip[:, j - 1] = np.where(f == 0, 1.0, f)
        for kd, _, i, t, h, s in (row for row in narr if row[0] == 3 and row[1] == j):
            Hk = quad(i, t, h)
            test(s * Hk[:, j - 1] > 0, np.abs(Hk[:, j - 1]) / np.maximum(np.abs(Hk).sum(1), 1e-300))
    for kd, j, i, t, h, s in (row for row in narr if row[0] in (1, 2)):
        a = np.abs(quad(i, t, h)); o = np.delete(a, j - 1, axis=1)
        rhs = (o.max(1) if o.shape[1] else np.zeros(n)) if kd == 1 else o.sum(1)
        test(a[:, j - 1] > rhs, np.abs(a[:, j - 1] - rhs) / np.maximum(a.sum(1), 1e-300))
    return ok, flip, margin


def omega_sim(cOm, narr, r, n_sim, seed, mid, s0=0, s1=None):
    """(n_ok, n_close) over simulations s0 .. s1 - 1 (default 0 .. n_sim - 1): those satisfying every row, and those whose
    decision margin is below 1e-9.  cOm(i) -> (H, r) array of c_{i,l} omega_k.  A simulation's outcome depends on its index
    alone, so counts over ranges add up."""
    ps, pos = periods(narr)
    nP = len(ps)
    s1 = n_sim if s1 is None else s1
    n_sim = s1 - s0
    s = np.arange(s0, s1, dtype=np.uint64)
    e = (s[:, None, None] * np.uint64(nP) + np.arange(nP, dtype=np.uint64)[None, :, None]) * np.uint64(r) + \
        np.arange(r, dtype=np.uint64)[None, None, :]
    E = rng_normal(seed, mid, RNG_NARR, e.ravel()).reshape(n_sim, nP, r)
    ok = np.ones(n_sim, bool); close = np.zeros(n_sim, bool)
    for kd, j, i, t, h, sg in narr:
        if kd == 0:
            v = sg * E[:, pos[t], j - 1]
            ok &= v > 0; close |= np.abs(v) < 1e-9
            continue
        cw = cOm(i)
        Hk = sum(cw[l][None, :] * E[:, pos[t + h - l], :] for l in range(h + 1))       # (n_sim, r)
        a = np.abs(Hk); scl = np.maximum(a.sum(1), 1e-300)
        if kd == 3:
            v = sg * Hk[:, j - 1]
            ok &= v > 0; close |= np.abs(v) / scl < 1e-9
        else:
            o = np.delete(a, j - 1, axis=1)
            rhs = (o.max(1) if o.shape[1] else np.zeros(n_sim)) if kd == 1 else o.sum(1)
            ok &= a[:, j - 1] > rhs; close |= np.abs(a[:, j - 1] - rhs) / scl < 1e-9
    return int(ok.sum()), int(close.sum())


def identify(Lam, R, A, Q, F, p, rows, narr, H, n_shock, n_rot, n_keep, n_sim, seed=0, mid=0, scale=None, batch=0):
    """dfm_narrative_sign_restrictions on one model: sign_oracle.identify's dict plus n_ok, weight (n_keep,), eps (n_keep, Tp,
    n_shock), n_close (simulations within 1e-9 of a decision, per slot) and margin over every candidate's decisions.  batch > 0
    decides the candidates `batch` at a time with decide_batch (for n_rot in the millions)."""
    Lam = np.asarray(Lam, float); R = np.asarray(R, float); F = np.asarray(F, float)
    N, r = Lam.shape; Tp = F.shape[0]
    out = dict(n_accept=0, cand=np.full(n_keep, -1), rot=np.full((n_keep, r, r), np.nan), resp=np.full((n_keep, N, H, n_shock), np.nan),
               fevd=np.full((n_keep, N, H, n_shock), np.nan), status=0, margin=np.inf, n_ok=np.zeros(n_keep, np.int64),
               weight=np.full(n_keep, np.nan), eps=np.full((n_keep, Tp, n_shock), np.nan), n_close=np.zeros(n_keep, np.int64))
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
    if np.isnan(F).any():
        out["status"] = 3
        return out
    if any(kd != 0 and not inm[i] for kd, j, i, t, h, s in narr):
        out["status"] = 1
        return out
    U = shocks_u(A, Q, F, p)
    C = SO.row_vectors(Lam, A, Q, p, rows, H) if rows else np.zeros((0, r))
    sign_shocks = [j for i, h, j, s in rows]
    c_of = lambda i: np.einsum("a,hab->hb", Lam[i], P)
    acc = []
    if batch:
        for c0 in range(0, n_rot, batch):
            Om = SO.omegas(seed, mid, np.arange(c0, min(n_rot, c0 + batch)), r)
            ok, flip, m = decide_batch(Om, C, sign_shocks, narr, c_of, U, n_shock)
            out["margin"] = min(out["margin"], float(m.min()))
            acc += [(c0 + c, flip[c]) for c in np.flatnonzero(ok)]
        Om = SO.omegas(seed, mid, [c for c, _ in acc[:n_keep]], r)
    else:
        Om = SO.omegas(seed, mid, np.arange(n_rot), r)
        for c in range(n_rot):
            ok, flip, m = decide(Om[c], C, sign_shocks, narr, c_of, U, n_shock)
            out["margin"] = min(out["margin"], m)
            if ok:
                acc.append((c, flip))
    out["n_accept"] = len(acc)
    kept = acc[:n_keep]
    if not kept:
        return out
    out["cand"][:len(kept)] = [c for c, _ in kept]
    Omk = np.array([(Om[q] if batch else Om[c]) * f[None, :] for q, (c, f) in enumerate(kept)])
    out["rot"][:len(kept)] = Omk
    out["resp"][:len(kept)], out["fevd"][:len(kept)] = SO.rotated_responses(Lam, R, P, Omk, n_shock, scale)
    out["eps"][:len(kept)] = np.einsum("ta,nak->ntk", U, Omk[:, :, :n_shock])
    for q, om in enumerate(Omk):
        if narr:
            n_ok, n_close = omega_sim(lambda i: c_of(i) @ om, narr, r, n_sim, seed, mid)
        else:
            n_ok, n_close = n_sim, 0
        out["n_ok"][q], out["n_close"][q] = n_ok, n_close
        out["weight"][q] = n_sim / n_ok if n_ok else np.inf
    return out


def _grid(w):
    """Positive finite doubles w -> Python integers on the common grid 2^e0 of the smallest one (exact)."""
    mant, ex = np.frexp(w)
    M = (mant * 2.0 ** 53).astype(np.int64)
    E = ex.astype(np.int64) - 53
    e0 = int(E.min())
    return [int(a) << int(b - e0) for a, b in zip(M, E)]


def weighted_percentiles(recs, w, q, near=False):
    """Per column, over the records with a non-NaN value and 0 < w < Inf, sorted by value: the first record i with
    100 sum_{j <= i} w_j >= q sum_j w_j in exact arithmetic (numpy's inverted_cdf rule with weights, without its rounding of the
    cumulative weights and of q / 100).
    near=True returns (lo, hi): the values of the records allowed when the sums are rounded, the exact record's sorted
    neighbours whose decision lies within 2^-100 sum_j w_j of the threshold (lo = hi = the exact record elsewhere)."""
    recs = np.asarray(recs, float); w = np.asarray(w, float)
    out = np.full((len(q), recs.shape[1]), np.nan)
    lo, hi = out.copy(), out.copy()
    qr = [(a, 100 * b) for a, b in (float(x).as_integer_ratio() for x in q)]      # q / 100 = a / b exactly
    for e in range(recs.shape[1]):
        ok = ~np.isnan(recs[:, e]) & (w > 0) & np.isfinite(w)
        if not ok.any():
            continue
        x = recs[ok, e]
        o = np.argsort(x, kind="stable")
        xs = x[o]
        cum = list(itertools.accumulate(_grid(w[ok][o])))
        T, m = cum[-1], len(cum)
        for k, (a, b) in enumerate(qr):
            # cum_i >= (a / b) T  <=>  b cum_i >= a T
            i = min(_first(cum, a * T, b), m - 1)
            out[k, e] = xs[i]
            if near:
                # |cum - (a / b) T| <= 2^-100 T  <=>  2^100 |b cum - a T| <= b T
                il = i - 1 if i > 0 and (a * T - b * cum[i - 1]) << 100 <= b * T else i
                ih = i + 1 if i + 1 < m and (b * cum[i] - a * T) << 100 <= b * T else i
                lo[k, e], hi[k, e] = xs[il], xs[ih]
    return (lo, hi) if near else out


def _first(cum, t, b):
    """The first i with b cum_i >= t (cum nondecreasing; len(cum) when none)."""
    lo_, hi_ = 0, len(cum)
    while lo_ < hi_:
        mid = (lo_ + hi_) // 2
        if b * cum[mid] >= t:
            hi_ = mid
        else:
            lo_ = mid + 1
    return lo_
