"""GeoGuessr metrics on the GPU (pigeon_b200.metrics, csrc/geo_metrics.cu) against the exact host oracle
(tests/metrics_oracle.py) and the reference golden (tests/golden/metrics.npz).

Country location must match the oracle exactly (country, nearest-fallback flag, pred_inside) on a synthetic world with
concave polygons, enclaves, islands, shared borders, an overlapping pair and a ring of 200 000 vertices, queried on
vertices, on edges, one ulp off edges, on rays through vertices and far outside.  The per-sample distance metrics are
exact wherever the oracle's decision margin exceeds 1e-9 relative (DESIGN.md §4's refiner-tie convention)."""
import json
import os

import numpy as np
import pytest
import torch

import metrics_oracle as mo
from pigeon_b200 import config, metrics
from pigeon_b200._lib import PigeonB200Error, check, current_stream_ptr, load, ptr

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "metrics.npz")
CASES = ("f32_1d_month", "f64_2d_yfcc", "f64_1d_no_mt")
MARGIN = 1e-9


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(GOLDEN))


def _case(g, name):
    p = f"{name}/in/"
    return {k[len(p):]: v for k, v in g.items() if k.startswith(p)}


def big_world(golden):
    """The golden world plus a 200 000-vertex ring (a noisy circle around (60, 40), dyadic radii) with a hole."""
    w = json.loads(golden["world"].tobytes().decode())
    n = 200_000
    t = np.linspace(0, 2 * np.pi, n, endpoint=False)
    rng = np.random.default_rng(7)
    rad = 8 + np.round(rng.normal(0, 0.05, n) * 1024) / 1024
    ring = np.stack([60 + rad * np.cos(t), 40 + rad * np.sin(t)], 1)
    ring = np.concatenate([ring, ring[:1]])
    hole = [[58, 38], [58, 42], [62, 42], [62, 38], [58, 38]]
    w["features"].append({"type": "Feature", "properties": {"name": "Big"},
                          "geometry": {"type": "Polygon", "coordinates": [ring.tolist(), hole]}})
    return w


def queries(verts, ring_off, rng):
    """Points on vertices, on edge midpoints (exact for dyadic edges), one ulp off both, on rays through vertices,
    random points, and points outside everything (one with an exact nearest tie between West and East)."""
    edges = np.setdiff1d(np.arange(len(verts) - 1), ring_off[1:] - 1)
    pick = rng.choice(edges, 300, replace=False)
    small = edges[edges < ring_off[-3]]                               # every edge but the big ring's and its hole's
    pick = np.concatenate([pick, small])
    on_vert = verts[pick]
    mid = (verts[pick] + verts[pick + 1]) / 2
    pts = [on_vert, mid]
    for base in (on_vert, mid):
        for dx, dy in ((1, 0), (-1, 0), (0, 1), (0, -1)):
            pts.append(np.stack([np.nextafter(base[:, 0], base[:, 0] + dx * np.inf) if dx else base[:, 0],
                                 np.nextafter(base[:, 1], base[:, 1] + dy * np.inf) if dy else base[:, 1]], 1))
    ray = verts[pick].copy()
    ray[:, 0] -= rng.uniform(0.1, 5, len(ray))                         # horizontal ray through a vertex
    pts.append(ray)
    pts.append(rng.uniform([-15, -15], [75, 55], (1500, 2)))
    pts.append(np.array([[5, 17], [5, -3], [-20, 40], [11, 11], [40, 0], [100, 100], [-100, -60], [31, 31], [17, 9]],
                        dtype=np.float64))
    return np.concatenate(pts)


@pytest.fixture(scope="module")
def world(golden, cuda):
    w = big_world(golden)
    csr = metrics.parse_geojson(w)
    idx = metrics.CountryIndex(*csr)
    geoms = mo.geometries_from_csr(*csr[:4])
    return w, csr, idx, geoms


def test_locate_matches_exact_oracle(world):
    _, csr, idx, geoms = world
    rng = np.random.default_rng(3)
    labels = queries(csr[0], csr[1], rng)
    preds = np.concatenate([labels[1:], labels[:1]])
    country, flags, inside = (t.cpu().numpy() for t in idx.locate(labels, preds))
    oc, of, oi = mo.locate(geoms, labels, preds)
    bad = np.flatnonzero((country != oc) | (flags != of) | (inside != oi))
    assert bad.size == 0, [(labels[i].tolist(), country[i], oc[i], flags[i], of[i], inside[i], oi[i]) for i in bad[:10]]
    assert of.sum() > 10 and oi.sum() > 100 and (oi == 0).sum() > 100
    tie = np.flatnonzero((labels == [5, 17]).all(1))[0]
    assert country[tie] == 4 and flags[tie] == 1          # West and East are both exactly 1 away: the lower index wins
    assert country[labels.tolist().index([14.0, 2.0])] == 1  # a vertex of Holland's hole and of the enclave


def test_index_and_locate_are_deterministic(world):
    _, csr, idx, _ = world
    idx2 = metrics.CountryIndex(*csr)
    assert torch.equal(idx._index, idx2._index) and torch.equal(idx._entries, idx2._entries)
    lab = np.random.default_rng(4).uniform([-15, -15], [75, 55], (5000, 2))
    a = [t.cpu() for t in idx.locate(lab, lab[::-1].copy())]
    b = [t.cpu() for t in idx2.locate(lab, lab[::-1].copy())]
    assert all(torch.equal(x, y) for x, y in zip(a, b))


def _scalers(golden, tmp_path, monkeypatch):
    import joblib
    from sklearn.preprocessing import StandardScaler
    for which, attr in (("main", "SCALER_PATH"), ("yfcc", "SCALER_PATH_YFCC")):
        ms = golden[f"scaler_{which}"]
        sc = StandardScaler()
        sc.mean_, sc.scale_, sc.var_, sc.n_features_in_ = ms[:6], ms[6:], ms[6:] ** 2, 6
        joblib.dump(sc, str(tmp_path / which))
        monkeypatch.setattr(config, attr, str(tmp_path / which))


def _results(c):
    g = c.get
    return (g("predictions"), g("cell_preds"), g("preds_mt"), g("preds_climate"), g("preds_month"), g("top5"),
            g("labels"), g("cell_labels"), g("labels_mt"), g("labels_climate"), g("labels_month"))


def _check_distances(d, ref, preds, labels):
    """float32 predictions: 1e-6 relative (numpy's float32 cos is not correctly rounded).  float64: 8 ulp, widened by the
    condition number kappa of asin(sqrt(a)) in the haversine term a, which amplifies last-bit differences of sin / cos
    toward antipodal pairs (kappa >= 1/2, growing without bound as a -> 1).  Two libms meet here: CUDA's fp64 sin, cos
    and asin are accurate to 2 ulp, numpy's to about 1, so a few ulp of `a` and of asin may differ on each side; 4 ulp,
    the budget of one library, was exceeded (6 ulp, one sample in 100 003) on the first H100 run."""
    if preds.dtype == np.float32:
        np.testing.assert_allclose(d, ref, rtol=1e-6, atol=1e-9)
        return
    a = np.clip(mo.haversine_a(preds, np.asarray(labels, dtype=np.float64)), 1e-300, 1 - 1e-16)
    kappa = np.sqrt(a) / (2 * np.sqrt(1 - a) * np.arcsin(np.sqrt(a)))
    ulps = np.abs(d - ref) / np.spacing(np.abs(ref))
    bound = 8 * np.maximum(1.0, 2 * kappa)
    assert np.all(ulps <= bound), (ulps.max(), (ulps / bound).max())


def _mean_rtol(preds):
    return 1e-6 if preds.dtype == np.float32 else 1e-13


def _low_margin_share(ref_d):
    """Share of samples whose margin is within MARGIN (< 1 %): each Under_*_km share may differ by at most that, and the
    mean score by at most that many points."""
    low = mo.margins(ref_d) <= MARGIN
    assert low.mean() < 0.01
    return low.mean()


@pytest.mark.parametrize("name", CASES)
def test_compute_metrics_matches_reference_golden(golden, name, cuda, tmp_path, monkeypatch):
    _scalers(golden, tmp_path, monkeypatch)
    c = _case(golden, name)
    idx = metrics.CountryIndex(golden["verts"], golden["ring_off"], golden["part_ring_off"], golden["geom_part_off"])
    out = metrics.compute_geoguessr_metrics(_results(c), countries=idx)
    keys, vals = list(golden[f"{name}/keys"]), golden[f"{name}/values"]
    assert list(out) == keys
    res, dist, (country, flags, inside) = metrics.geo_metrics(c["predictions"], c["labels"], c["cell_preds"],
                                                              c["cell_labels"] if c["cell_labels"].ndim == 1 else
                                                              np.argmax(c["cell_labels"], -1), c["top5"], idx)
    d = dist.cpu().numpy()
    _check_distances(d, golden[f"{name}/distances"], c["predictions"], c["labels"])
    np.testing.assert_array_equal(country.cpu().numpy(), golden[f"{name}/country"])
    np.testing.assert_array_equal(inside.cpu().numpy(), golden[f"{name}/pred_inside"])
    slack = _low_margin_share(golden[f"{name}/distances"])
    got = np.asarray([float(v) for v in out.values()])
    np.testing.assert_allclose(got[0], vals[0], rtol=_mean_rtol(c["predictions"]))
    assert got[1] == np.median(d)
    np.testing.assert_allclose(got[1], vals[1], rtol=1e-6 if c["predictions"].dtype == np.float32 else 1e-15)
    assert np.all(np.abs(got[2:12] - vals[2:12]) <= slack) and abs(got[13] - vals[13]) <= slack
    assert np.array_equal(got[[12, 14, 15]], vals[[12, 14, 15]])
    np.testing.assert_array_equal(got[16:], vals[16:])


@pytest.mark.parametrize("f32", [False, True])
def test_metrics_kernel_against_oracle_at_scale(cuda, f32):
    rng = np.random.default_rng(11 + f32)
    N, C, k = 100_003, 3000, 5
    labels = rng.uniform([-180, -90], [180, 90], (N, 2))
    preds = labels + rng.normal(0, 1, (N, 2)) * rng.choice([1e-4, 1e-2, 0.1, 1, 5, 30], N)[:, None]
    preds = preds.astype(np.float32) if f32 else preds
    cl = rng.integers(0, C, N)
    cp = np.where(rng.random(N) < 0.3, cl, rng.integers(0, C, N))
    topk = rng.integers(0, C, (N, k))
    hit = rng.random(N) < 0.4
    topk[hit, 2] = cl[hit]
    w = {"type": "FeatureCollection", "features": [{"type": "Feature", "properties": {}, "geometry": {
        "type": "Polygon", "coordinates": [[[-180, -90], [0, -90], [0, 90], [-180, 90], [-180, -90]]]}}]}
    idx = metrics.CountryIndex(*metrics.parse_geojson(w))
    res, dist, (_, _, inside) = metrics.geo_metrics(preds, labels, cp, cl, topk, idx)
    d = dist.cpu().numpy()
    ref, ref_d = mo.metrics(preds, labels, cp, cl, topk, inside.cpu().numpy())
    _check_distances(d, ref_d, preds, labels)
    low = mo.margins(ref_d) <= MARGIN
    assert low.mean() < 0.01
    ok = ~low
    for t, km in enumerate(mo.KM):
        assert np.array_equal(d[ok] < km, ref_d[ok] < km)
    assert np.array_equal(mo.scores(d[ok]), mo.scores(ref_d[ok]))
    vals = np.asarray(list(ref.values()))
    np.testing.assert_allclose(res[0], vals[0], rtol=_mean_rtol(preds))
    np.testing.assert_allclose(res[0], np.mean(d), rtol=1e-13)
    assert res[1] == np.median(d)
    slack = low.sum() / N
    assert np.all(np.abs(res[2:12] - vals[2:12]) <= slack) and abs(res[13] - vals[13]) <= slack
    assert res[12] == vals[12] and res[14] == vals[14] and res[15] == vals[15]
    assert 0.2 < res[12] < 0.8
    # run to run: identical bits
    res2, dist2, _ = metrics.geo_metrics(preds, labels, cp, cl, topk, idx)
    assert np.array_equal(res.view(np.uint64), res2.view(np.uint64)) and torch.equal(dist, dist2)
    # odd and even N: np.median semantics
    for n in (1, 2, 7, 10):
        r, dd, _ = metrics.geo_metrics(preds[:n], labels[:n], cp[:n], cl[:n], topk[:n], idx)
        assert r[1] == np.median(dd.cpu().numpy())


def test_bad_arguments(golden, cuda):
    idx = metrics.CountryIndex(golden["verts"], golden["ring_off"], golden["part_ring_off"], golden["geom_part_off"])
    p = np.zeros((4, 2))
    ones = np.zeros(4, np.int64)
    with pytest.raises(ValueError, match="shape"):
        metrics.geo_metrics(np.zeros((4, 3)), p, ones, ones, ones.reshape(4, 1), idx)
    with pytest.raises(ValueError, match="inconsistent"):
        metrics.geo_metrics(p, p, ones[:3], ones, ones.reshape(4, 1), idx)
    with pytest.raises(ValueError, match="finite"):
        metrics.geo_metrics(np.array([[0, np.nan]] * 4), p, ones, ones, ones.reshape(4, 1), idx)
    with pytest.raises(ValueError, match="finite"):
        metrics.geo_metrics(p, np.array([[np.inf, 0]] * 4), ones, ones, ones.reshape(4, 1), idx)
    with pytest.raises(ValueError, match="inconsistent"):
        metrics.geo_metrics(p[:0], p[:0], ones[:0], ones[:0], ones[:0].reshape(0, 1), idx)
    lib = load()
    dev = torch.device("cuda")
    t = lambda a: torch.as_tensor(a).to(dev)
    x, i, tk, ins = t(p), t(ones), t(ones.reshape(4, 1)), t(np.zeros(4, np.uint8))
    d, res = torch.empty(4, dtype=torch.float64, device=dev), torch.empty(16, dtype=torch.float64, device=dev)
    need = int(lib.pg_geo_metrics_workspace_bytes(4))
    ws = torch.empty(need, dtype=torch.uint8, device=dev)
    with pytest.raises(PigeonB200Error, match="too small"):
        check(lib.pg_geo_metrics(ptr(x), 0, ptr(x), 4, ptr(i), ptr(i), ptr(tk), 1, ptr(ins), ptr(ws), need - 1, ptr(d),
                                 ptr(res), current_stream_ptr()), "pg_geo_metrics")
    with pytest.raises(PigeonB200Error, match="bad sizes"):
        check(lib.pg_geo_metrics(ptr(x), 0, ptr(x), 4, ptr(i), ptr(i), ptr(tk), 0, ptr(ins), ptr(ws), need, ptr(d),
                                 ptr(res), current_stream_ptr()), "pg_geo_metrics")
    small = metrics.PgCountries.from_buffer_copy(idx._c)
    small.index_bytes = 16
    with pytest.raises(PigeonB200Error, match="too small"):
        check(lib.pg_country_locate(small, ptr(x), ptr(x), 4, None, None, None, current_stream_ptr()), "pg_country_locate")
    with pytest.raises(ValueError, match="offsets"):
        metrics.CountryIndex(golden["verts"], golden["ring_off"][:-1], golden["part_ring_off"], golden["geom_part_off"])


def test_evaluate_model_with_metrics(golden, cuda, tmp_path, monkeypatch):
    """evaluate_model(..., partial(compute_geoguessr_metrics, countries=idx), ..., refiner) returns -Geocell_accuracy and
    passes the metrics the same results a direct call computes."""
    from functools import partial
    from pigeon_b200 import ProtoRefiner, SuperGuessr
    from pigeon_b200.loops import evaluate_model
    z = np.load(os.path.join(os.path.dirname(__file__), "golden", "refiner_count1.npz"))
    bank = {k[5:]: z[k] for k in z.files if k.startswith("bank_")}
    D, C = bank["proto_emb"].shape[1], int(bank["cell_off"].shape[0]) - 1
    g = torch.Generator().manual_seed(5)
    n = 37
    emb = torch.randn(n, 4, D, generator=g) * 0.3
    labels = torch.rand(n, 2, generator=g, dtype=torch.float64) * 30
    labels_clf = torch.randint(0, C, (n,), generator=g)

    class DS(torch.utils.data.Dataset):
        def __len__(self):
            return n

        def __getitem__(self, i):
            if isinstance(i, str):
                return {"labels": labels.numpy(), "labels_clf": labels_clf.numpy()}[i]
            return dict(embedding=emb[i], labels=labels[i], labels_clf=labels_clf[i])

    cells = np.stack([np.linspace(-170, 170, C), np.linspace(-80, 80, C)], 1)
    sg = SuperGuessr(None, panorama=True, num_candidates=10, embed_dim=D, geocells=cells).to(cuda).eval()
    ref = ProtoRefiner(topk=5, max_refinement=1e6, temperature=1.6, protos=bank).eval()
    idx = metrics.CountryIndex(golden["verts"], golden["ring_off"], golden["part_ring_off"], golden["geom_part_off"])
    seen = []

    def fn(results):
        seen.append(results)
        return metrics.compute_geoguessr_metrics(results, countries=idx)

    class Args:
        per_device_eval_batch_size = 16

    ret = evaluate_model(sg, DS(), fn, Args(), ref)
    direct = metrics.compute_geoguessr_metrics(seen[0], countries=idx)
    assert seen[0][0].dtype == np.float32
    assert ret == -direct['Geocell_accuracy']
    again = evaluate_model(sg, DS(), partial(metrics.compute_geoguessr_metrics, countries=idx), Args(), ref)
    assert again == ret
    assert list(direct)[:16] == list(golden["f64_1d_no_mt/keys"])
