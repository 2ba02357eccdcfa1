"""CPU-only: the Python layer of narrative sign restrictions.  The defaults of api.narrative_identified_set and
api.narrative_restricted_responses lie within their bounds, and the history bands of narrative_identified_set (historical
decompositions of the rotated models, through the HOST-EMULATION build of the kernel source) give the spec's contributions."""
import inspect
import os
import sys
import types

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "emu"))
import build_emu  # noqa: E402
import identified_oracle as IO  # noqa: E402
import narrative_oracle as NO  # noqa: E402
import sign_checks as SC  # noqa: E402
import sign_oracle as SO  # noqa: E402
from dynamic_factor_models_b200 import Library, api  # noqa: E402


@pytest.fixture(scope="module")
def lib():
    L = Library(build_emu.build())
    yield L
    L.close()


def _defaults(f):
    return {k: v.default for k, v in inspect.signature(f).parameters.items() if v.default is not inspect.Parameter.empty}


def test_defaults_within_bounds():
    d = _defaults(api.narrative_restricted_responses)
    assert 1 <= d["n_chain"] * d["n_keep"] * d["rot_per_draw"] <= 16384
    assert 1 <= _defaults(api.narrative_identified_set)["n_keep"] <= 16384
    # the bound check passes with the defaults: the call goes on to the model (which has no EM estimates here)
    m = types.SimpleNamespace(em=None)
    with pytest.raises(Exception) as ei:
        api.narrative_restricted_responses(m, [], [("shock", 1, 5, 1)], 4)
    assert "rot_per_draw" not in str(ei.value)


def test_history_is_the_rotated_decomposition(lib):
    """_narr_history's contrib at base row t0 is xstd_i H_{i,k}(t0 + 1, h) at row t0 + 1 + h for every kept draw, and rest
    + contrib adds up to the contributions of all r shocks; the bands are the weighted percentiles of the draws."""
    r, p, N, Tp, H = 3, 2, 7, 14, 4
    Lam, R, A, Q, sc = SC.models(r, p, N, 1, seed=8)
    Lam, R, A, Q = Lam[0], R[0], A[0], Q[0]
    Lam[5] = np.nan
    F = np.random.default_rng(2).standard_normal((Tp, r))
    rot = SO.omegas(4, 0, np.arange(6), r) * np.array([1.0, -1.0, 1.0])[None, None, :]
    w = np.array([1.0, 2.5, np.inf, 1.2, 4.0, 1.0])
    b = dict(em=dict(A=A, Q=Q, R=R), Lam=Lam, Xs=np.zeros((Tp, N)), xstd=sc)
    q = np.array([5.0, 50.0, 95.0])
    row0 = 4
    out = api._narr_history(lib, b, F, row0, rot, w, 2, q, True)
    U = NO.shocks_u(A, Q, F, p)
    P = IO.psi(A, Q, p, Tp)
    for n in range(len(rot)):
        for i in (0, 3, N - 1):
            for h in (0, 2, Tp - row0 - 2):
                Hk = NO.contributions(Lam[i] @ P, rot[n], U, row0 + 1, h) * sc[i]
                got = out["contrib_draws"][n, i, row0 + 1 + h]
                np.testing.assert_allclose(got, Hk[:2], rtol=1e-10, atol=1e-12 * np.abs(Hk).max())
                np.testing.assert_allclose(out["rest_draws"][n, i, row0 + 1 + h], Hk[2:].sum(), rtol=1e-9, atol=1e-12 * np.abs(Hk).max())
    assert np.isnan(out["contrib_draws"][:, 5]).all() and np.isnan(out["contrib_bands"][:, 5]).all()
    ok = np.isfinite(w)
    ref = NO.weighted_percentiles(out["contrib_draws"].reshape(len(rot), -1), np.where(ok, w, 0.0), q)
    np.testing.assert_array_equal(out["contrib_bands"].reshape(len(q), -1), ref)
