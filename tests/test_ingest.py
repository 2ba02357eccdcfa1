"""Product-side panel ingestion (dynamic_factor_models_b200/ingest.py, SURVEY 8(f)2) against the committed output of
the ingestion oracle (tests/golden/hom_fac_1_panels.npz = oracle/readin.py on the reference's workbook).  The workbook
tests read an .xlsx rebuilt from tests/golden/hom_fac_1_workbook.npz.xz: the exact cell values of the reference's
data/hom_fac_1.xlsx that the ingestion reads (see tests/golden/make_golden.py)."""
import io
import lzma
import os
import zipfile
from xml.sax.saxutils import escape

import numpy as np
import pytest

from dynamic_factor_models_b200 import ingest

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
SHEETS = ("Monthly", "Quarterly")
_MAIN = "http://schemas.openxmlformats.org/spreadsheetml/2006/main"


def _sheet_cells(z, sheet):
    """(row, col) -> str or float of one sheet, decoded from the fixture (inverse of make_golden.workbook_fixture)."""
    names, codes, scales = z[f"{sheet}_names"], z[f"{sheet}_codes"], z[f"{sheet}_scales"]
    ns, ncodes = len(names), codes.shape[0]
    missing = np.unpackbits(z[f"{sheet}_missing"], axis=1)[:, :ns + 1].astype(bool)         # (periods, 1 + ns), column 0: dates
    zz = z[f"{sheet}_ints"].T.copy().view(np.uint64).ravel()
    ints = (zz >> np.uint64(1)).astype(np.int64) ^ -(zz & np.uint64(1)).astype(np.int64)  # undo the zig-zag code
    raw = z[f"{sheet}_raw"].T.copy().view(np.float64).ravel()
    cells = {(0, 1 + j): str(n) for j, n in enumerate(names)}
    cells.update({(3 + i, 1 + j): float(codes[i, j]) for i in range(ncodes) for j in range(ns)})
    head, ki, kr = 3 + ncodes, 0, 0
    for c in range(ns + 1):
        rows = np.flatnonzero(~missing[:, c])
        if scales[c] >= 0:
            vals = np.cumsum(ints[ki:ki + len(rows)]) / 10.0 ** scales[c]
            ki += len(rows)
        else:
            vals = raw[kr:kr + len(rows)]
            kr += len(rows)
        cells.update({(head + r, c): float(v) for r, v in zip(rows, vals)})
    return cells


def _col(c):
    s = ""
    c += 1
    while c:
        c, m = divmod(c - 1, 26)
        s = chr(65 + m) + s
    return s


def _sheet_xml(cells):
    rows = {}
    for (r, c), v in sorted(cells.items()):
        ref = f"{_col(c)}{r + 1}"
        rows.setdefault(r, []).append(f'<c r="{ref}" t="inlineStr"><is><t>{escape(v)}</t></is></c>' if isinstance(v, str)
                                      else f'<c r="{ref}"><v>{v!r}</v></c>')
    body = "".join(f'<row r="{r + 1}">{"".join(cs)}</row>' for r, cs in sorted(rows.items()))
    return f'<?xml version="1.0" encoding="UTF-8"?><worksheet xmlns="{_MAIN}"><sheetData>{body}</sheetData></worksheet>'


@pytest.fixture(scope="module")
def XLSX(tmp_path_factory):
    """The workbook rebuilt from the fixture: the Monthly and Quarterly sheets as a minimal .xlsx."""
    with open(os.path.join(GOLDEN, "hom_fac_1_workbook.npz.xz"), "rb") as f:
        z = np.load(io.BytesIO(lzma.decompress(f.read())))
    path = str(tmp_path_factory.mktemp("workbook") / "hom_fac_1.xlsx")
    rel = "http://schemas.openxmlformats.org/officeDocument/2006/relationships"
    with zipfile.ZipFile(path, "w", zipfile.ZIP_DEFLATED) as w:
        w.writestr("[Content_Types].xml",
                   '<?xml version="1.0" encoding="UTF-8"?><Types xmlns="http://schemas.openxmlformats.org/package/2006/content-types">'
                   '<Default Extension="xml" ContentType="application/xml"/>'
                   '<Override PartName="/xl/workbook.xml" ContentType="application/vnd.openxmlformats-officedocument.spreadsheetml.sheet.main+xml"/>'
                   + "".join(f'<Override PartName="/xl/worksheets/sheet{i + 1}.xml" '
                             'ContentType="application/vnd.openxmlformats-officedocument.spreadsheetml.worksheet+xml"/>' for i in range(len(SHEETS)))
                   + "</Types>")
        w.writestr("xl/workbook.xml", f'<?xml version="1.0" encoding="UTF-8"?><workbook xmlns="{_MAIN}" xmlns:r="{rel}"><sheets>'
                   + "".join(f'<sheet name="{s}" sheetId="{i + 1}" r:id="rId{i + 1}"/>' for i, s in enumerate(SHEETS)) + "</sheets></workbook>")
        w.writestr("xl/_rels/workbook.xml.rels",
                   '<?xml version="1.0" encoding="UTF-8"?><Relationships xmlns="http://schemas.openxmlformats.org/package/2006/relationships">'
                   + "".join(f'<Relationship Id="rId{i + 1}" Type="{rel}/worksheet" Target="worksheets/sheet{i + 1}.xml"/>'
                             for i in range(len(SHEETS))) + "</Relationships>")
        for i, s in enumerate(SHEETS):
            w.writestr(f"xl/worksheets/sheet{i + 1}.xml", _sheet_xml(_sheet_cells(z, s)))
    return path


@pytest.mark.parametrize("datatype,key", [("All", "all"), ("Real", "real")])
def test_readin_data_matches_oracle_fixture(XLSX, panels, datatype, key):
    p = ingest.readin_data(XLSX, datatype)
    gold = panels[f"{key}_bpdata"]
    assert p.bpdata.shape == gold.shape
    assert (np.isnan(p.bpdata) == np.isnan(gold)).all()
    np.testing.assert_allclose(p.bpdata, gold, rtol=1e-11, atol=1e-13)      # biweight sums are associated differently
    np.testing.assert_array_equal(p.inclcode, panels[f"{key}_inclcode"])
    assert p.bpnamevec == [str(n) for n in panels[f"{key}_names"]]
    assert p.calds == [tuple(int(v) for v in r) for r in panels["calds"]]
    assert p.row(1959, 3) == 3 and p.row(2014, 4) == 224                   # Stock_Watson.ipynb:1266-1267


def test_survey_panel_facts(XLSX):
    """SURVEY.md section 8: 224 x 207, N = 139 estimation series, 94.3 % observed, 94 balanced columns."""
    p = ingest.readin_data(XLSX, "All")
    est = p.bpdata[2:224][:, p.inclcode == 1]
    assert p.bpdata.shape == (224, 207) and est.shape == (222, 139)
    assert abs(1 - np.isnan(est).mean() - 0.943) < 5e-4
    assert int((~np.isnan(est).any(0)).sum()) == 94


def test_transform_and_biweight_small():
    x = np.array([1.0, 2.0, 4.0, 8.0, np.nan, 32.0])
    np.testing.assert_allclose(ingest.transform_series(x, 5)[1:4], np.log(2) * np.ones(3))
    assert np.isnan(ingest.transform_series(x, 6)[:2]).all()
    X = np.column_stack([np.arange(10.0), np.r_[np.nan, np.ones(9)]])
    tr = ingest.biweight_trend(X, 4.0)
    assert np.isnan(tr[0, 1]) and np.allclose(tr[1:, 1], 1.0)              # local mean of a constant is the constant
    assert np.allclose(tr[4:6, 0], X[4:6, 0])                              # symmetric window around an interior point of a line


def test_workbook_to_table2B_through_product_code(XLSX, notebook_tables):
    """Workbook -> product ingestion -> estimate_factor! through the kernel source (host emulation build) ->
    golden Table 2B row r = 8 (trace R2 0.501, BN-ICp2 -0.223; Stock_Watson.ipynb:619-628)."""
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(__file__), "emu"))
    import build_emu
    import dynamic_factor_models_b200 as D
    lib = D.Library(build_emu.build())
    try:
        p = ingest.readin_data(XLSX, "All")
        m = D.DFMModel(p.bpdata, p.inclcode, 20, 40, p.row(1959, 3), p.row(2014, 4), 0, 8, 1e-8, 4, 4)
        D.estimate_factor(m, lib=lib)
        gold = np.array(notebook_tables["table2B"])[7]                  # nfac, traceR2, margR2, BN-ICp2, AH-ER
        assert abs((1 - m.fes.ssr / m.fes.tss) - gold[1]) < 6e-4
        assert abs(D.bai_ng_criterion(m) - gold[3]) < 6e-4
    finally:
        lib.close()
