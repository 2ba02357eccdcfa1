"""CPU oracle for the dynamic-factor-model hot path.  TEST INFRASTRUCTURE ONLY.

Nothing under ``oracle/`` is shipped or measured as product: only ``tests/``,
``__graft_entry__.smoke()`` and ``bench.py``'s ``cpu_baseline`` / ``--impl
reference`` legs may import it, and there only as the checker or the timed CPU
baseline.  The product path (``dynamic_factor_models_b200``) never imports it and
fails loudly when its CUDA library is missing.

Modules
-------
xlsx_min   stdlib-only .xlsx reader (stands in for ExcelReaders.readxlsheet)
readin     restatement of the reference's readin_functions.jl  (panel ingestion)
dfm_ref    restatement of the reference's dfm_functions.ipynb  (PCA / ALS "EM" /
           loadings / factor VAR / IRF / constraints / Bai-Ng / Amengual-Watson)
           -- PINNED against the golden tables stored in Stock_Watson.ipynb
kalman_em  FP64 Kalman filter + RTS smoother + EM for the state-space DFM.
           The reference has NO such code (``struct Parametric`` is an empty
           placeholder, dfm_functions.ipynb:23) => PARITY UNPINNED for this part:
           this file *is* the spec; it is checked by invariants only.
dgp        frozen synthetic data generator (SURVEY.md section 8d)
c/         plain-C port of kalman_em + ALS used as the timed CPU baseline
"""
