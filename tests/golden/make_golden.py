"""Generate the committed fixtures under tests/golden/ from a checkout of QuantEcon/dynamic_factor_models.
Usage:  python tests/golden/make_golden.py REFERENCE_DIR

Writes
  hom_fac_1_panels.npz   output of the ingestion oracle (oracle/readin.py) on
                         REFERENCE_DIR/data/hom_fac_1.xlsx for datatype :All and :Real
                         (the notebook's `dataset_all` / `dataset`, Stock_Watson.ipynb:160,180)
  notebook_tables.json   the numeric tables stored as cell outputs of Stock_Watson.ipynb
                         (Tables 2A, 2B, 2C, 3 (visible part), 4, 5) -- the reference's only
                         golden values (SURVEY.md section 4)
  hom_fac_1_workbook.npz.xz  the cells of the workbook's Monthly and Quarterly sheets that the
                         ingestion reads (names, code rows, dates, data of every series it uses;
                         exact doubles), from which tests/test_ingest.py rebuilds an .xlsx
"""
import io, json, lzma, os, re, sys
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", ".."))
from oracle.readin import readin_data  # noqa: E402
from oracle.xlsx_min import read_sheet  # noqa: E402

# sheet name -> (number of series, number of code rows, number of data rows); readin_functions.jl:258-283
SHEETS = {"Monthly": (148, 6, 672), "Quarterly": (85, 5, 224)}
# series that the ingestion looks up by name whatever their inclusion code (deflators, Kilian's index)
BY_NAME = {"GLOBAL_ACT", "PCEPI", "PCEPILFE", "PCECTPI", "JCXFE", "GDPCTPI"}


def workbook_fixture(xlsx):
    """Compact, exact copy of the cells the ingestion reads.  Per sheet: series names, code rows, and the data block
    (dates in column 0).  Series with inclusion code 0 that are not looked up by name are left out (blank).  A data column
    whose values are all k / 10^d for integers k (d <= 9) is stored as the differences of k with its d; the other columns
    as raw doubles; both byte-plane shuffled, then the whole archive is xz-compressed."""
    arrays = {}
    for sheet, (ns, ncodes, nobs) in SHEETS.items():
        g = read_sheet(xlsx, sheet)
        head = 3 + ncodes
        names = [str(v) for v in g[0][1:ns + 1]]
        codes = np.array([[float(v) for v in g[3 + i][1:ns + 1]] for i in range(ncodes)])
        incl = codes[ncodes - 2]
        D = np.array([[v if isinstance(v, float) else np.nan for v in (row + [None] * (ns + 1))[:ns + 1]] for row in g[head:head + nobs]])
        for j in range(ns):
            if incl[j] == 0 and names[j].upper() not in BY_NAME:
                D[:, j + 1] = np.nan
        scales, ints, raw = [], [], []
        for c in range(ns + 1):
            v = D[~np.isnan(D[:, c]), c]
            d = next((d for d in range(10) if np.array_equal(np.round(v * 10.0 ** d) / 10.0 ** d, v)), -1)
            scales.append(d)
            if d >= 0:
                ints.append(np.diff(np.round(v * 10.0 ** d).astype(np.int64), prepend=0))
            else:
                raw.append(v)
        k = np.concatenate(ints)
        zz = ((k << 1) ^ (k >> 63)).astype(np.uint64)                     # zig-zag: small magnitudes -> small codes
        arrays.update({f"{sheet}_names": np.array(names), f"{sheet}_codes": codes, f"{sheet}_missing": np.packbits(np.isnan(D), axis=1),
                       f"{sheet}_scales": np.array(scales, np.int8),
                       f"{sheet}_ints": zz.view(np.uint8).reshape(-1, 8).T.copy(),
                       f"{sheet}_raw": np.concatenate(raw).view(np.uint8).reshape(-1, 8).T.copy()})
    buf = io.BytesIO()
    np.savez(buf, **arrays)
    return lzma.compress(buf.getvalue(), preset=9 | lzma.PRESET_EXTREME)

ANSI = re.compile(r"\x1b\[[0-9;]*m")


def parse_millboard(text):
    rows = []
    for line in ANSI.sub("", text).splitlines():
        cells = [c.strip() for c in line.strip().strip("|").split("|")]
        try:
            vals = [float(c) for c in cells[1:]]
        except ValueError:
            continue
        if vals:
            rows.append(vals)
    return rows


def main(REF):
    xlsx = os.path.join(REF, "data", "hom_fac_1.xlsx")
    a = readin_data(xlsx, "All"); r = readin_data(xlsx, "Real")
    np.savez_compressed(os.path.join(HERE, "hom_fac_1_panels.npz"),
                        all_bpdata=a["bpdata"], all_inclcode=a["inclcode"], all_names=np.array(a["bpnamevec"]),
                        real_bpdata=r["bpdata"], real_inclcode=r["inclcode"], real_names=np.array(r["bpnamevec"]),
                        calds=np.array(a["calds"]))
    nb = json.load(open(os.path.join(REF, "Stock_Watson.ipynb")))
    outs = {}
    for i, c in enumerate(nb["cells"]):
        if c["cell_type"] != "code":
            continue
        txt = []
        for o in c.get("outputs", []):
            if "text" in o:
                txt.append("".join(o["text"]))
            elif "data" in o and "text/plain" in o["data"]:
                txt.append("".join(o["data"]["text/plain"]))
        outs[i] = txt
    tables = {}
    tables["table2A"] = parse_millboard(outs[35][0])      # cols: nfac, traceR2, margR2, BN-ICp2, AH-ER
    tables["table2B"] = parse_millboard(outs[37][0])
    tables["table2C"] = parse_millboard(outs[39][0])      # rows: n dynamic; cols: n dyn, then static 1..10
    # Table 3: 207x10 R2, visible: first 13 + last 12 rows, columns 1-3 and 8-10
    t3 = []
    for line in outs[55][0].splitlines()[1:]:
        toks = line.replace("…", " ").replace("⋱", " ").replace("⋮", " ").split()
        if len(toks) == 6:
            t3.append([float(x) for x in toks])
    tables["table3_visible"] = {"rows_head": 13, "rows_tail": 12, "cols": [1, 2, 3, 8, 9, 10], "values": t3}
    nums = lambda s: [[float(x) for x in ln.split()] for ln in s.splitlines()[1:] if ln.strip()]
    tables["table4"] = {"chow_qlr_r4": nums(outs[58][0]), "chow_qlr_r8": nums(outs[58][1]),
                        "cor_r4": nums(outs[58][2]), "cor_r8": nums(outs[58][3])}
    t5 = {}
    lines = outs[61][0].splitlines()
    for k in range(0, len(lines), 3):
        name = lines[k].split()[1]
        t5[name] = {"resid": [float(x) for x in lines[k + 1].strip("[]").split()],
                    "level": [float(x) for x in lines[k + 2].strip("[]").split()]}
    tables["table5"] = t5
    tables["source"] = "stored cell outputs of the reference's Stock_Watson.ipynb (Julia 1.0.2)"
    json.dump(tables, open(os.path.join(HERE, "notebook_tables.json"), "w"), indent=1)
    with open(os.path.join(HERE, "hom_fac_1_workbook.npz.xz"), "wb") as f:
        f.write(workbook_fixture(xlsx))
    print({k: (len(v) if isinstance(v, list) else "...") for k, v in tables.items()})


if __name__ == "__main__":
    main(sys.argv[1])
