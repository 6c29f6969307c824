"""The host build of the fire-weather device code under AddressSanitizer + UBSan (every fixture case and the
longest rings).  Run from the repository root:

    LD_PRELOAD=$(g++ -print-file-name=libasan.so) ASAN_OPTIONS=detect_leaks=0 python tools/fwi_host_asan.py
"""
import sys, os
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for d in (os.path.join(ROOT, "tests"), ROOT, os.path.join(ROOT, "tests", "golden")):
    sys.path.insert(0, d)
import numpy as np
import fwi_host_build as hb
import host_build
hb.load = lambda: host_build.load("fwi_asan", "fwi_host.cpp", signatures=hb.SIGNATURES,
                                  flags=("-O1", "-g", "-fsanitize=address,undefined", "-fno-omit-frame-pointer"))
import make_golden as mg
from test_fire_oracle import case_inputs, check_outputs
g = np.load(os.path.join(ROOT, "tests", "golden", "ref_cffwis.npz"))
for name in mg.CFFWIS_CASES:
    args, kw, exp = case_inputs(g, name)
    got = hb.run(*args, **kw)
    check_outputs(got, exp, name, exact_frac=0.99)
    print(name, "ok")
# extreme parameters: longest rings
inp = mg.cffwis_inputs(seed=5, C=16, T=400)
tc = lambda a: np.ascontiguousarray(a.T)
base = (tc(inp["tas"]), tc(inp["pr"]), tc(inp["hurs"]), tc(inp["ws"]), tc(inp["snd"]), inp["mth"], inp["lat"])
nanv = np.full(16, np.nan, np.float32)
hb.run(*base, None, nanv, nanv, nanv, np.zeros(16, np.float32), outputs=["DC","DMC","FFMC","season_mask"], season_method="GFWED",
       dry_start="GFWED+SNOW", temp_condition_days=32, snow_condition_days=32, snow_cover_days=128)
hb.run(*base, None, nanv, nanv, nanv, np.zeros(16, np.float32), outputs=["DC","season_mask"], season_method="GFWED",
       temp_condition_days=1, snow_condition_days=1, snow_cover_days=1, dry_start="GFWED+SNOW")
print("extremes ok")
