"""Restatement of the reference's readin_functions.jl (panel ingestion).  ORACLE ONLY.

Missing values are NaN.  Every function cites the reference lines it follows.
Needs the reference's data/hom_fac_1.xlsx; its OUTPUT for the two notebook
configurations is committed under tests/golden/ by tests/golden/make_golden.py so
that the tests do not need the workbook.
"""
import numpy as np
from .xlsx_min import read_sheet, excel_serial_to_ymd


def n_periods(initvec, lastvec, per_year):
    """MonthlyData / QuarterlyData constructors, readin_functions.jl:29-36."""
    return per_year * (lastvec[0] - initvec[0] - 1) + lastvec[1] + (per_year - initvec[1] + 1)


def transform(x, tcode):
    """readin_functions.jl:105-115 (tcode 1..6)."""
    x = np.asarray(x, float)
    if tcode == 1:
        return x.copy()
    if tcode == 2:
        return np.concatenate([[np.nan], x[1:] - x[:-1]])
    if tcode == 3:
        return np.concatenate([[np.nan, np.nan], x[2:] - 2 * x[1:-1] + x[:-2]])
    if tcode == 4:
        return np.log(x)
    if tcode == 5:
        return transform(np.log(x), 2)
    if tcode == 6:
        return transform(np.log(x), 3)
    raise ValueError(tcode)


def adjust_outlier(x, outliercode, io_method):
    """readin_functions.jl:127-198.  In place on x (1-D float array with NaN)."""
    if outliercode == 0:
        return
    thr = {1: 4.5, 2: 3.0}[outliercode]                       # :128-132
    obs = x[~np.isnan(x)]
    zm = np.median(obs)                                       # :137
    iqr = np.quantile(obs, 0.75) - np.quantile(obs, 0.25)     # :138 (Julia default = type 7)
    ya = np.abs(x - zm)
    with np.errstate(invalid="ignore"):
        i_out = ya > thr * iqr                                # NaN compares False
    idx = np.flatnonzero(i_out)
    if io_method == 0:                                        # :152-155
        x[idx] = np.nan
    elif io_method == 1:                                      # :159-164
        sgn = (x[idx] > 0).astype(float) - (x[idx] < 0).astype(float)
        x[idx] = zm + sgn * (thr * iqr)
    elif io_method == 2:                                      # :168-171
        x[idx] = zm
    elif io_method == 3:                                      # :175-184 local median +-3
        for i in idx:
            w = x[max(0, i - 3):min(len(x), i + 4)]
            x[i] = np.median(w[~np.isnan(w)])
    elif io_method == 4:                                      # :188-198 one-sided median, 5 preceding
        for i in idx:
            w = x[max(0, i - 5):i + 1]
            x[i] = np.median(w[~np.isnan(w)])
    else:
        raise ValueError(io_method)


def bi_weight_filter(y, weight):
    """readin_functions.jl:335-348: local biweight-kernel mean ignoring missing."""
    T = len(y)
    trend = np.full(T, np.nan)
    obs = ~np.isnan(y)
    tt = np.arange(1, T + 1, dtype=float)
    yo = y[obs]
    for t in np.flatnonzero(obs):
        dt = (tt - (t + 1)) / weight
        w = 15.0 / 16.0 * (1 - dt ** 2) ** 2
        w[np.abs(dt) >= 1] = 0.0
        wo = w[obs]
        wo = wo / wo.sum()
        trend[t] = np.dot(wo, yo)
    return trend


def _read_block(xlsx, sheet, ndesc, ncodes, dnobs, ns, monthly, datatype,
                correct_outlier=True, io_method=4, cat_include=(1, 2, 3, 5)):
    """readin_monthly_data, readin_functions.jl:206-253 (+ headers :258-283)."""
    grid = read_sheet(xlsx, sheet)
    nhead = 1 + ndesc + ncodes
    rows = grid[:nhead + dnobs]
    main = [r[1:ns + 1] + [None] * (ns - len(r[1:ns + 1])) for r in rows]
    dates = [excel_serial_to_ymd(r[0]) for r in rows[nhead:]]
    names = [str(s).upper() for s in main[0]]
    if monthly:                                               # :258-270
        tcode = [int(v) for v in main[4]]; defcode = [int(v) for v in main[5]]
        outl = [int(v) for v in main[6]]; incl = [int(v) for v in main[7]]
        cat = [float(v) for v in main[8]]
    else:                                                     # :272-283
        tcode = [int(v) for v in main[3]]; defcode = [int(v) for v in main[4]]
        outl = [int(v) for v in main[5]]; incl = [int(v) for v in main[6]]
        cat = [float(v) for v in main[7]]
    dm = np.array([[v if isinstance(v, float) else np.nan for v in r] for r in main[nhead:]], float)
    # deflators :285-301
    if monthly:
        pdef = dm[:, names.index("PCEPI")].copy(); plfe = dm[:, names.index("PCEPILFE")].copy(); pgdp = None
        j = names.index("GLOBAL_ACT")                          # standardize_killian! :306-313
        col = dm[:, j]; ok = ~np.isnan(col)
        dm[ok, j] = (col[ok] - col[ok].mean()) / col[ok].std(ddof=1)
    else:
        pdef = dm[:, names.index("PCECTPI")].copy(); plfe = dm[:, names.index("JCXFE")].copy()
        pgdp = dm[:, names.index("GDPCTPI")].copy()
    incl = np.array(incl); cat = np.array(cat)
    if datatype == "Real":                                    # :254-256
        used = (incl != 0) & np.isin(np.floor(cat), cat_include)
    else:
        used = incl != 0
    ui = np.flatnonzero(used)
    data = dm[:, ui].copy()
    for k, j in enumerate(ui):                                # deflate_series! :40-76
        dc = defcode[j]
        if dc == 1: data[:, k] = data[:, k] / pdef
        elif dc == 2: data[:, k] = data[:, k] / plfe
        elif dc == 3: data[:, k] = data[:, k] / pgdp
    if monthly:                                               # monthly_to_quarterly :83-100
        yq = [(y, (m + 2) // 3) for (y, m, _) in dates]
        uq = sorted(set(yq))
        dq = np.full((len(uq), data.shape[1]), np.nan)
        yq_arr = np.array([uq.index(v) for v in yq])
        for t in range(len(uq)):
            dq[t] = data[yq_arr == t].mean(axis=0)             # NaN if any month missing
        data, dates_q = dq, uq
    else:
        dates_q = [(y, (m + 2) // 3) for (y, m, _) in dates]
    raw = data.copy()
    with np.errstate(invalid="ignore", divide="ignore"):
        for k, j in enumerate(ui):                            # transform! :117-125
            data[:, k] = transform(data[:, k], tcode[j])
    noa = data.copy()
    if correct_outlier:
        for k, j in enumerate(ui):                            # :247
            adjust_outlier(data[:, k], outl[j], io_method)
    return dict(data=data, raw=raw, noa=noa, dates=dates_q, cat=cat[ui], incl=incl[ui],
                names=[names[j] for j in ui])


def readin_data(xlsx, datatype="All", biweight=100.0,
                m_init=(1959, 1), m_last=(2014, 12), m_ns=148,
                q_init=(1959, 1), q_last=(2014, 4), q_ns=85):
    """readin_data, readin_functions.jl:355-382 with the notebook's arguments
    (Stock_Watson.ipynb:143-144, :160/:180)."""
    m = _read_block(xlsx, "Monthly", 2, 6, n_periods(m_init, m_last, 12), m_ns, True, datatype)
    q = _read_block(xlsx, "Quarterly", 2, 5, n_periods(q_init, q_last, 4), q_ns, False, datatype)
    assert m["dates"] == q["dates"]
    cat = np.concatenate([m["cat"], q["cat"]])
    order = np.argsort(cat, kind="stable")                    # sortperm :368 (ties by index)
    bpdata = np.hstack([m["data"], q["data"]])[:, order]
    unfiltered = bpdata.copy()
    trend = np.full_like(bpdata, np.nan)
    if biweight is not None:                                  # detrend_var! :317-324
        for i in range(bpdata.shape[1]):
            trend[:, i] = bi_weight_filter(bpdata[:, i], biweight)
            bpdata[:, i] = bpdata[:, i] - trend[:, i]
    names = (m["names"] + q["names"])
    return dict(bpdata=bpdata, bpdata_unfiltered=unfiltered, bpdata_trend=trend,
                bpdata_raw=np.hstack([m["raw"], q["raw"]])[:, order],
                bpdata_noa=np.hstack([m["noa"], q["noa"]])[:, order],
                bpcatcode=cat[order], inclcode=np.concatenate([m["incl"], q["incl"]])[order],
                bpnamevec=[names[i] for i in order], calds=m["dates"],
                calvec=np.array([y + (qq - 1) / 4 for (y, qq) in m["dates"]]))


def find_row_number(date, calds):
    """dfm_functions.ipynb:555-556 (1-based row of (year, quarter))."""
    return calds.index(tuple(date)) + 1
