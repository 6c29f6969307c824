"""GPU: the fire-weather kernel (xc_fwi_f32) through the C ABI against the reference fixtures, the oracle and
through the host layer.  A looser share of bit-identical values is asked for than on the CPU: CUDA's float64 exp /
log / pow differ from glibc's by an ulp now and then, which flips a float32 rounding that the recurrences then
carry for days; every value must still agree to 2e-6.  The kernel's device code is also verified on the CPU as a
host build (tests/test_fire_host_core.py)."""
import numpy as np
import pytest

from oracle import fire_oracle as FO
from test_fire_oracle import case_inputs, check_outputs, golden, mg  # noqa: F401

pytestmark = pytest.mark.gpu


def run_on_device(args, kw):
    import torch

    from xclim_b200 import device
    tas, pr, hurs, ws, snd, mth, lat, mask, dc0, dmc0, ffmc0, wpr = args
    outputs = kw["outputs"]
    over = {k: v for k, v in kw.items() if k != "outputs"}
    from xclim_b200.fire import default_params
    p = {k: (v if not isinstance(v, tuple) else v[0]) for k, v in default_params.items()}
    p.update({k: v for k, v in over.items() if k in p})
    dry = over.get("dry_start")
    P = device.fwi_params(over.get("season_method"), over.get("overwintering", False), dry,
                          over.get("initial_start_up", True), **p)
    d = lambda a, dt=torch.float32: None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to("cuda", dt)  # noqa: E731
    res = device.fire_weather(d(tas), d(pr), d(hurs), d(ws), d(snd), mth, lat, d(mask, torch.uint8), d(dc0), d(dmc0),
                              d(ffmc0), d(wpr), outputs, P)
    torch.cuda.synchronize()
    return {k: (v.cpu().numpy().astype(bool) if k == "season_mask" else v.cpu().numpy()) for k, v in res.items()}


def test_elementwise_kernel_on_device(cuda, golden):  # noqa: F811
    import torch

    from test_fire_oracle import assert_index_close
    from xclim_b200 import device
    g = golden
    d = lambda a: torch.from_numpy(np.ascontiguousarray(a.T)).cuda()   # noqa: E731
    ffmc, dmc, dc = (d(g[f"always_on__{k}"]) for k in ("FFMC", "DMC", "DC"))
    assert_index_close(device.fire_elementwise("ISI", d(g["ws"]), ffmc).cpu().numpy(), g["always_on__ISI"].T, "ISI")
    assert_index_close(device.fire_elementwise("BUI", dmc, dc).cpu().numpy(), g["always_on__BUI"].T, "BUI")
    assert_index_close(device.fire_elementwise("FWI", d(g["always_on__ISI"]), d(g["always_on__BUI"])).cpu().numpy(),
                       g["always_on__FWI"].T, "FWI")
    assert_index_close(device.fire_elementwise("DSR", d(g["always_on__FWI"])).cpu().numpy(), g["always_on__DSR"].T, "DSR")
    got = device.fire_elementwise("OWDC", torch.tensor([300.0, 100.0, 1.0], device="cuda"),
                                  torch.tensor([110.0, 50.0, 550.0], device="cuda"), (0.75, 0.75, 15))
    np.testing.assert_allclose(got.cpu().numpy(), [109.4657, 105.176, 15.0], rtol=1e-6)


@pytest.mark.parametrize("name", list(mg.CFFWIS_CASES))
def test_kernel_matches_reference_fixture(cuda, golden, name):  # noqa: F811
    args, kw, exp = case_inputs(golden, name)
    got = run_on_device(args, kw)
    check_outputs(got, exp, name, exact_frac=0.90)


def test_kernel_matches_oracle_on_a_wider_grid(cuda):
    """1500 cells (several CTAs, a ragged last one), 3 years, all latitude bands."""
    rng = np.random.default_rng(21)
    base = mg.cffwis_inputs(seed=31, C=16, T=1095)
    reps = 94
    C = 16 * reps - 4
    tile = lambda a: np.ascontiguousarray(np.tile(a, (reps, 1))[:C].T)   # noqa: E731  (T, C)
    tas, pr, hurs, ws, snd = (tile(base[k]) for k in ("tas", "pr", "hurs", "ws", "snd"))
    tas = (tas + rng.normal(0, 1.5, tas.shape)).astype(np.float32)
    pr = (pr * rng.uniform(0.5, 1.5, pr.shape)).astype(np.float32)
    lat = rng.uniform(-90, 90, C)
    dc0 = rng.uniform(20, 500, C).astype(np.float32)
    dc0[::7] = np.nan
    nanv = np.full(C, np.nan, np.float32)
    for kw in (dict(season_method=None, outputs=["DC", "DMC", "FFMC", "ISI", "BUI", "FWI", "DSR"]),
               dict(season_method="GFWED", dry_start="GFWED+SNOW", snow_cover_days=45, snow_min_mean_depth=0.03,
                    outputs=["DC", "DMC", "FFMC", "ISI", "BUI", "FWI", "season_mask"]),
               dict(season_method="LA08", overwintering=True, outputs=["DC", "season_mask", "winter_pr"])):
        args = (tas, pr, hurs, ws, snd, base["mth"], lat, None, dc0, nanv, nanv, np.zeros(C, np.float32))
        exp = FO.fire_weather_calc(*args, **kw)
        got = run_on_device(args, kw)
        check_outputs(got, {k: np.asarray(v) for k, v in exp.items()}, str(kw), exact_frac=0.90)


def test_host_layer_on_device(cuda):
    from test_fire_host_layer import check_bodies
    from xclim_b200 import Field, fire
    check_bodies(fire, Field)


def test_fire_weather_streams_from_files_on_device(cuda, tmp_path):
    from test_fire_host_layer import check_streaming
    check_streaming(tmp_path)



def test_kernel_every_mode_combination_against_the_oracle(cuda):
    """All season x overwintering x dry-start x initial_start_up combinations with random parameters: the kernel
    against the oracle, which tests/test_fire_host_core.py pins to the reference on the SAME combinations
    (there, with the host build of this kernel's device code)."""
    import itertools
    rng = np.random.default_rng(123)
    T = 320
    n = 0
    for trial, (season, ow, dry, isu) in enumerate(itertools.product(
            [None, "mask", "WF93", "LA08", "GFWED"], [False, True], [None, "CFS", "GFWED", "GFWED+SNOW"], [True, False])):
        if ow and season is None:
            continue
        inp = mg.cffwis_inputs(seed=1000 + trial, C=16, T=T)
        dc0, dmc0, ffmc0, wpr = mg.cffwis_state(inp, [None, "some", "all"][trial % 3])
        over = dict(season_method=season, overwintering=ow, dry_start=dry, initial_start_up=isu,
                    temp_condition_days=int(rng.integers(1, 6)), snow_condition_days=int(rng.integers(1, 6)),
                    snow_cover_days=int(rng.integers(5, 70)), temp_start_thresh=float(rng.uniform(8, 14)),
                    temp_end_thresh=float(rng.uniform(2, 7)), snow_thresh=float(rng.choice([0.01, 0.03])),
                    prec_thresh=float(rng.choice([1.0, 2.5])), dc_dry_factor=int(rng.integers(2, 7)),
                    dmc_dry_factor=int(rng.integers(1, 4)), snow_min_cover_frac=float(rng.uniform(0.3, 0.8)),
                    snow_min_mean_depth=float(rng.uniform(0.02, 0.1)), carry_over_fraction=float(rng.choice([0.5, 0.75, 1.0])),
                    wetting_efficiency_fraction=float(rng.choice([0.5, 0.75, 0.9])))
        outs = ["DC", "DMC", "FFMC", "ISI", "BUI", "FWI", "DSR"]
        mask = None
        if season == "mask":
            m = np.zeros((16, T), bool)
            st = rng.random(16) < 0.5
            for t in range(T):
                st = np.where(rng.random(16) < 0.03, ~st, st)
                m[:, t] = st
            mask = np.ascontiguousarray(m.T)
        elif season is not None:
            outs.append("season_mask")
        if ow:
            outs.append("winter_pr")
        tc = lambda a: np.ascontiguousarray(a.T)   # noqa: E731
        args = (tc(inp["tas"]), tc(inp["pr"]), tc(inp["hurs"]), tc(inp["ws"]), tc(inp["snd"]), inp["mth"], inp["lat"], mask,
                dc0, dmc0, ffmc0, wpr)
        exp = FO.fire_weather_calc(*args, outputs=outs, **over)
        got = run_on_device(args, dict(outputs=outs, **over))
        check_outputs(got, {k: np.asarray(v) for k, v in exp.items()}, f"{season},{ow},{dry},{isu}", exact_frac=0.90)
        n += 1
    assert n == 72


def test_kernel_branch_point_inputs_against_the_oracle(cuda):
    """The branch-point inputs of tests/test_fire_host_core.py::test_branch_point_inputs_against_the_reference
    (there: oracle and host build against the reference), here the kernel against the oracle."""
    rng = np.random.default_rng(7)
    C, T = 32, 240
    f32 = lambda a: np.ascontiguousarray(a, dtype=np.float32)   # noqa: E731
    for trial in range(6):
        tas = rng.choice([-45.0, -2.8, -1.1, 0.0, 21.1, 35.0, 50.0], size=(C, T)) + rng.normal(0, 0.5, (C, T))
        pr = rng.choice([0.0, 0.5, 0.50001, 1.5, 1.50001, 2.8, 2.80001, 50.0, 300.0], size=(C, T))
        hurs = rng.choice([0.0, 1e-3, 5.0, 50.0, 99.999, 100.0], size=(C, T))
        ws = rng.choice([0.0, 1e-3, 10.0, 100.0, 250.0], size=(C, T))
        snd = rng.choice([0.0, 0.01, 0.010001, 0.5], size=(C, T))
        if trial % 3 == 0:
            for a in (tas, pr, hurs, ws):
                a[rng.random((C, T)) < 0.002] = np.nan
        mth = rng.integers(1, 13, T).astype(np.int64)
        lat = rng.choice([-90, -30, -15, 15, 30, 90, -29.999, 14.999, 0], size=C).astype(np.float64)
        dc0, dmc0, ffmc0, wpr = mg.cffwis_state({"tas": f32(tas)}, [None, "some", "all"][trial % 3])
        if trial % 3:
            dc0[:4], dmc0[:4], ffmc0[:4] = [0.0, 1e-3, 800.0, 2000.0], [0.0, 33.0, 65.0, 500.0], [0.0, 101.0, 50.0, 99.9]
        for season, ow, dry in ((None, False, None), ("WF93", True, "CFS"), ("GFWED", False, "GFWED+SNOW"), ("LA08", True, None)):
            outs = ["DC", "DMC", "FFMC", "ISI", "BUI", "FWI", "DSR"] + (["season_mask"] if season else []) + \
                (["winter_pr"] if ow else [])
            over = dict(season_method=season, overwintering=ow, dry_start=dry, snow_cover_days=10)
            args = tuple(f32(a.T) for a in (tas, pr, hurs, ws, snd)) + (mth, lat, None, dc0, dmc0, ffmc0, wpr)
            exp = FO.fire_weather_calc(*args, outputs=outs, **over)
            got = run_on_device(args, dict(outputs=outs, **over))
            check_outputs(got, {k: np.asarray(v) for k, v in exp.items()}, f"{trial} {season}", exact_frac=0.90)
