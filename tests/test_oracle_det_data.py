"""oracle/det_data_cpu.py (the numpy restatement of the two VoteNet detection `__getitem__`s) against the original: bit for bit under
the same draws, against tests/golden/det_data.npz and, where oracle/det_data_ref.py staged it, against the original run live."""
import os

import numpy as np
import pytest

from oracle import det_data_cpu as O

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "det_data.npz")
NUM_POINTS = 200
SCANNET = ("scene0000_00", "scene0001_00", "scene0002_00")
SUNRGBD = ("000001", "000002", "000003")


@pytest.fixture(scope="module")
def golden():
    with np.load(GOLDEN) as z:
        return {k: z[k] for k in z.files}


def cases(g, prefix):
    return sorted({k.split("/")[0] for k in g if k.startswith(prefix)})


def draws_of(g, case):
    kinds = list(g[f"{case}/draw_kinds"])
    return [(str(k), g[f"{case}/draw{i}"]) for i, k in enumerate(kinds)]


def replay(record):
    it = iter(record)

    def draws(kind, *a, **kw):
        k, v = next(it)
        assert k == kind, (k, kind)
        return v[()] if v.ndim == 0 else v.copy()
    return draws


def scannet_config():
    from oracle import det_data_ref
    mods = det_data_ref.load()
    return None if mods is None else mods[0].DC


def sunrgbd_config():
    from oracle import det_data_ref
    mods = det_data_ref.load()
    return None if mods is None else mods[1].DC


def parse(case):
    parts = case.split("_")
    opt = {p[0]: bool(int(p[1:])) for p in parts[2:]}
    return int(parts[1]), opt


def oracle_item(g, case, dc, draws):
    s, opt = parse(case)
    if case.startswith("scannet"):
        n = SCANNET[s]
        return O.scannet_item(g[f"files/{n}_vert"], g[f"files/{n}_sem_label"], g[f"files/{n}_ins_label"], g[f"files/{n}_bbox"],
                              dc.nyu40ids, dc.mean_size_arr, NUM_POINTS, opt["h"], opt["a"], s, draws)
    n = SUNRGBD[s]
    return O.sunrgbd_item(g[f"files/{n}_pc/pc"], g[f"files/{n}_votes/point_votes"], g[f"files/{n}_bbox"], dc.num_heading_bin,
                          dc.mean_size_arr, NUM_POINTS, opt["c"], opt["h"], opt["a"], s, draws)


def assert_same(got, want):
    assert got.keys() == want.keys()
    for k in want:
        a, b = np.asarray(got[k]), np.asarray(want[k])
        assert a.dtype == b.dtype and a.shape == b.shape, k
        assert np.array_equal(a, b), k          # == : signed zeros of padded rows compare equal


@pytest.mark.parametrize("dataset", ["scannet", "sunrgbd"])
def test_restatement_matches_golden(golden, dataset):
    dc = scannet_config() if dataset == "scannet" else sunrgbd_config()
    if dc is None:
        pytest.skip("the original's dataset configs are not staged under oracle/_ref/")
    cs = cases(golden, dataset + "_")
    assert len(cs) == (12 if dataset == "scannet" else 24)
    for case in cs:
        want = {k.split("/", 1)[1]: golden[k] for k in golden if k.startswith(case + "/") and "draw" not in k}
        assert_same(oracle_item(golden, case, dc, replay(draws_of(golden, case))), want)


@pytest.mark.parametrize("dataset", ["scannet", "sunrgbd"])
def test_restatement_matches_live_original(golden, dataset, tmp_path):
    from oracle import det_data_ref
    mods = det_data_ref.load()
    if mods is None:
        pytest.skip("the original detection datasets are not staged under oracle/_ref/")
    from tests.golden.make_det_data_golden import write_scenes
    write_scenes(str(tmp_path))
    cls = mods[0].ScannetDetectionDataset if dataset == "scannet" else mods[1].SunrgbdDetectionVotesDataset
    dc = mods[0].DC if dataset == "scannet" else mods[1].DC
    for case in cases(golden, dataset + "_"):
        s, opt = parse(case)
        record = draws_of(golden, case)
        got = det_data_ref.item(cls, str(tmp_path), SCANNET if dataset == "scannet" else SUNRGBD, NUM_POINTS, opt.get("c", False),
                                opt["h"], opt["a"], s, replay(record))
        assert_same(oracle_item(golden, case, dc, replay(record)), got)


def test_scannet_quirk_cases_are_covered(golden):
    """The golden scenes hold instance 0, ids near 2^32, K = 0 and K = 64, N below and above num_points, and an instance whose first
    sampled row carries a non-object label while others of its rows carry object labels."""
    dc = scannet_config()
    ks = [len(golden[f"files/{n}_bbox"]) for n in SCANNET]
    ns = [len(golden[f"files/{n}_vert"]) for n in SCANNET]
    assert 0 in ks and 64 in ks and min(ns) < NUM_POINTS < max(ns)
    ins = np.concatenate([golden[f"files/{n}_ins_label"] for n in SCANNET])
    assert 0 in ins and ins.max() >= 2 ** 31
    if dc is None:
        return
    found = False
    for case in cases(golden, "scannet_"):
        s, _ = parse(case)
        n = SCANNET[s]
        ch = draws_of(golden, case)[0][1]
        sem, ins = golden[f"files/{n}_sem_label"][ch], golden[f"files/{n}_ins_label"][ch]
        for i in np.unique(ins):
            rows = np.flatnonzero(ins == i)
            obj = np.isin(sem[rows], dc.nyu40ids)
            found |= (not obj[0]) and obj.any()
    assert found
