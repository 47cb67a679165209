"""Valid-intrinsics regions on the GPU (csrc/regions.cu, csrc/uncertainty.cu, csrc/image_transforms.cu), against
numpy restatements written here and against the public pieces they are built from:

- the regional residual statistics against the reference's per-cell loop (mrcal/calibration.py:1800-1866), with
  outliers and corners put by hand on, just inside and just outside cell boundaries and off the imager;
- the uncertainty of several cameras from one factorization against projection_uncertainty() per camera, bit for bit;
- _compute_valid_intrinsics_region() against the same pipeline composed from numpy statistics,
  projection_uncertainty() and the host contour, and valid_intrinsics_regions() against it for every camera;
- is_within_valid_intrinsics_region() against a strict-interior restatement (edges and vertices are outside);
- a computed region driving image_transformation_map(mask_valid_intrinsics_region_from=True)."""
import numpy as np
import pytest

import mrcal_b200
from mrcal_b200 import regions, synthetic

pytestmark = pytest.mark.gpu

SPL = "LENSMODEL_SPLINED_STEREOGRAPHIC_order=3_Nx=11_Ny=8_fov_x_deg=150"
METHODS = ("mean-pcam", "cross-reprojection-rrp-Jfp", "cross-reprojection-ccp")


def _models(kw):
    return [mrcal_b200.cameramodel(optimization_inputs=kw, icam_intrinsics=i) for i in range(len(kw["intrinsics"]))]


def np_stats(kw, x, icam, gw, gh):
    """The reference's _report_regional_statistics() per-cell loop, restated"""
    W, H = kw["imagersizes"][icam]
    centers = mrcal_b200.sample_imager(gw, gh, W, H)
    rcell = np.array((float(W - 1) / (gw - 1), float(H - 1) / (gh - 1)), dtype=float) / 2.
    obs = kw["observations_board"]
    xb = x[:obs[..., 0].size * 2].reshape(obs.shape[:-1] + (2,))
    sel = np.ones(obs.shape[:-1], bool)
    sel[kw["indices_frame_camintrinsics_camextrinsics"][:, 1] != icam] = False
    sel[obs[..., 2] <= 0.] = False
    err, q = xb[sel], obs[sel][:, :2]
    out = np.zeros((gh, gw, 3))
    scale = np.zeros((gh, gw))
    for i in range(gh):
        for j in range(gw):
            idx = np.abs(q - centers[i, j]) < rcell
            e = err[idx[:, 0] * idx[:, 1]].ravel()
            out[i, j] = (0., 0., len(e)) if len(e) <= 5 else (np.mean(e), np.std(e), len(e))
            scale[i, j] = np.sqrt(np.mean(e * e)) if len(e) else 0.
    return out, scale


def _stats_problem(lensmodel, Ncameras, seed):
    kw, _ = synthetic.make_problem(lensmodel=lensmodel, Ncameras=Ncameras, Nframes=8, W=8, H=6, seed=seed,
                                   pixel_noise=0.3)
    obs = kw["observations_board"]
    rng = np.random.default_rng(seed)
    flat = obs.reshape(-1, 3)
    flat[rng.choice(flat.shape[0], flat.shape[0] // 10, replace=False), 2] = -1.   # outliers
    flat[rng.choice(flat.shape[0], 5, replace=False), 2] = 0.
    # corners exactly on, just inside and just outside cell boundaries, and off the imager
    W, H = kw["imagersizes"][0]
    gw, gh = 12, int(round(H / W * 12))
    c = mrcal_b200.sample_imager(gw, gh, W, H)
    r = np.array((float(W - 1) / (gw - 1), float(H - 1) / (gh - 1))) / 2.
    k = 0
    for (i, j) in ((2, 3), (3, 5), (4, 8), (1, 1)):
        for dx, dy in ((r[0], 0.), (-r[0], r[1]), (np.nextafter(r[0], 0), 0.), (0., -np.nextafter(r[1], 0)),
                       (np.nextafter(r[0], 1e9), np.nextafter(r[1], 1e9)), (r[0] * (1 - 1e-15), -r[1] * (1 - 1e-15))):
            flat[k, :2] = c[i, j] + (dx, dy)
            flat[k, 2] = 1.
            k += 7
    flat[k, :2] = (-50., 10.)
    flat[k + 3, :2] = (W + 3., H + 9.)
    return kw, gw, gh


@pytest.mark.parametrize("lensmodel,Ncameras", [("LENSMODEL_OPENCV8", 3), (SPL, 2), ("LENSMODEL_OPENCV8", 4)])
def test_regional_statistics(lensmodel, Ncameras):
    kw, gw, gh = _stats_problem(lensmodel, Ncameras, seed=11 + Ncameras)
    x = mrcal_b200.optimizer_callback(**kw, no_jacobian=True, no_factorization=True)[1]
    W, H = kw["imagersizes"][0]
    P = mrcal_b200.Problem(**kw)
    try:
        grids = [regions._cell_grid(kw["imagersizes"][i], gw, gh) for i in range(Ncameras)]
        args = (list(range(Ncameras)), np.array([g[0] for g in grids]), np.array([g[1] for g in grids]))
        stats, xd = P.regional_statistics(*args)
        stats2, _ = P.regional_statistics(*args)
    finally:
        P.close()
    assert np.array_equal(stats, stats2, equal_nan=True)             # fixed-order sums
    assert np.array_equal(xd, x)
    few = 0
    for icam in range(Ncameras):
        ref, scale = np_stats(kw, x, icam, gw, gh)
        assert np.array_equal(stats[icam, ..., 2], ref[..., 2])
        # the sums are in another order than numpy's: 1e-12 of the cell's rms residual (the mean of residuals that
        # cancel can be much smaller than they are)
        tol = 1e-12 * np.maximum(np.abs(ref[..., :2]), scale[..., None])
        assert (np.abs(stats[icam, ..., :2] - ref[..., :2]) <= tol).all()
        few += ((ref[..., 2] > 0) & (ref[..., 2] <= 5)).sum()
        # the public single-camera function agrees
        m = mrcal_b200.cameramodel(optimization_inputs=kw, icam_intrinsics=icam)
        mean, stdev, count, using = mrcal_b200._report_regional_statistics(m, gridn_width=gw)
        assert np.array_equal(np.stack((mean, stdev, count), -1), stats[icam])
        assert using == mrcal_b200.imagergrid_using((W, H), gw, gh)
    assert few > 0   # cells with at most 5 counts report (0, 0, count)


@pytest.fixture(scope="module")
def solved_opencv8():
    kw, _ = synthetic.make_problem(lensmodel="LENSMODEL_OPENCV8", Ncameras=3, Nframes=16, W=8, H=6, seed=4,
                                   pixel_noise=0.3)
    mrcal_b200.optimize(**kw)
    return kw


@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("distance", [None, 7.])
def test_uncertainty_cameras_bitwise(solved_opencv8, method, distance):
    kw = solved_opencv8
    models = _models(kw)
    rng = np.random.default_rng(2)
    ps = [rng.normal(0, 1, (n, 3)) + (0, 0, 4) for n in (37, 1, 90)]
    ps = [p / np.linalg.norm(p, axis=-1)[:, None] * (1. if distance is None else distance) for p in ps]
    atinf = distance is None
    P = mrcal_b200.Problem(**kw)
    try:
        Var, _ = P.projection_uncertainty_cameras(ps, [0, 1, 2], method=method, atinfinity=atinf)
        Var2, _ = P.projection_uncertainty_cameras([ps[2], ps[0]], [2, 0], method=method, atinfinity=atinf)
    finally:
        P.close()
    for i in range(3):
        ref = mrcal_b200.projection_uncertainty(ps[i], models[i], method=method, atinfinity=atinf)
        assert np.array_equal(Var[i], ref)
    assert np.array_equal(Var2[0], Var[2]) and np.array_equal(Var2[1], Var[0])


def _gap_threshold(v, quantile):
    """A threshold between two values of v near the given quantile, at least 1e-6 of their scale from both"""
    u = np.unique(np.asarray(v)[np.isfinite(v)])
    scale = max(np.abs(u).max(), 1e-300)
    gaps = np.flatnonzero(np.diff(u) > 1e-5 * scale)
    i = gaps[np.argmin(np.abs(gaps - quantile * len(u)))]
    return (u[i] + u[i + 1]) / 2.


def _pipeline(kw, model, thresholds, distance, gw):
    """_compute_valid_intrinsics_region() composed from public pieces and numpy"""
    lensmodel, intrinsics = model.intrinsics()
    W, H = model.imagersize()
    gh = int(round(H / W * gw))
    x = mrcal_b200.optimizer_callback(**kw, no_jacobian=True, no_factorization=True)[1]
    st, _ = np_stats(kw, x, model.icam_intrinsics(), gw, gh)
    q = mrcal_b200.sample_imager(gw, gh, W, H)
    v = mrcal_b200.unproject(q, lensmodel, intrinsics)
    v /= np.linalg.norm(v, axis=-1)[..., None]
    unc = mrcal_b200.projection_uncertainty(v if distance <= 0 else v * distance, model, atinfinity=distance <= 0,
                                            what="worstdirection-stdev")
    return st, unc, lambda t: regions._region_from_mask(
        regions._region_mask(lensmodel, st[..., 0], st[..., 1], st[..., 2], unc, *t), (W, H))


@pytest.mark.parametrize("lensmodel", ["LENSMODEL_OPENCV8", SPL])
@pytest.mark.parametrize("distance", [0., 5.])
def test_region_end_to_end(lensmodel, distance):
    kw, _ = synthetic.make_problem(lensmodel=lensmodel, Ncameras=2, Nframes=24, W=8, H=6, seed=8, pixel_noise=0.3)
    mrcal_b200.optimize(**kw)
    models = _models(kw)
    gw = 30
    for m in models:
        st, unc, pipeline = _pipeline(kw, m, None, distance, gw)
        t = (_gap_threshold(unc, 0.6), _gap_threshold(st[..., 0], 0.8), _gap_threshold(st[..., 1], 0.9), 3)
        ref = pipeline(t)
        r = mrcal_b200._compute_valid_intrinsics_region(m, *t, distance, gridn_width=gw)
        assert r.shape == ref.shape and np.array_equal(np.asarray(r, np.int32), np.asarray(ref, np.int32))


def test_region_of_centre_coverage():
    """Boards seen only in the middle of the imager: the region holds the centre and not the corners, and every
    camera's region from valid_intrinsics_regions() is what _compute_valid_intrinsics_region() gives it"""
    kw, _ = synthetic.make_problem(lensmodel="LENSMODEL_OPENCV8", Ncameras=3, Nframes=200, W=10, H=8, seed=5,
                                   pixel_noise=0.3)
    W, H = kw["imagersizes"][0]
    obs = kw["observations_board"]
    outside = (np.abs(obs[..., 0] - (W - 1) / 2.) > W * 0.3) | (np.abs(obs[..., 1] - (H - 1) / 2.) > H * 0.3)
    obs[..., 2][outside] = -1.
    # the boards mostly in the middle, and every frame's pose constrained by the corners left
    keep = (~outside).sum(axis=(1, 2)) >= outside[0].size // 2
    idx = kw["indices_frame_camintrinsics_camextrinsics"][keep]
    frames = np.unique(idx[:, 0])
    idx[:, 0] = np.searchsorted(frames, idx[:, 0])
    kw.update(indices_frame_camintrinsics_camextrinsics=np.ascontiguousarray(idx),
              observations_board=np.ascontiguousarray(obs[keep]), rt_ref_frame=np.ascontiguousarray(kw["rt_ref_frame"][frames]))
    assert all((idx[:, 1] == i).sum() >= 20 for i in range(3))
    mrcal_b200.optimize(**kw)
    parameters = (1, 0.5, 1.5, 3, 0)
    regs = mrcal_b200.valid_intrinsics_regions(kw, parameters)
    s = np.std(mrcal_b200.measurements_board(kw).ravel())
    for i, m in enumerate(_models(kw)):
        r = mrcal_b200._compute_valid_intrinsics_region(m, s, 0.5, 1.5 * s, 3, 0)
        assert np.array_equal(regs[i], r)
        assert r.shape[0] >= 4
        m.valid_intrinsics_region(r)
        inside = mrcal_b200.is_within_valid_intrinsics_region(
            np.array([[(W - 1) / 2., (H - 1) / 2.], [0., 0.], [W - 1., 0.], [0., H - 1.], [W - 1., H - 1.]]), m)
        assert inside.tolist() == [True, False, False, False, False]


def test_regions_refused_camera_warns(solved_opencv8, monkeypatch, capsys):
    """A camera whose grid cannot be unprojected gets None and the tool's warning; the others still get their region
    from the shared factorization"""
    kw = solved_opencv8
    good = mrcal_b200.valid_intrinsics_regions(kw)
    unproject = mrcal_b200.api.unproject

    def refuse_camera_1(q, lensmodel, intrinsics):
        if np.array_equal(intrinsics, kw["intrinsics"][1]):
            raise RuntimeError("camera 1 refused")
        return unproject(q, lensmodel, intrinsics)
    monkeypatch.setattr(mrcal_b200.api, "unproject", refuse_camera_1)
    regs = mrcal_b200.valid_intrinsics_regions(kw)
    err = capsys.readouterr().err
    assert regs[1] is None
    assert "WARNING: Couldn't compute valid-intrinsics region for camera 1" in err and "camera 1 refused" in err
    assert np.array_equal(regs[0], good[0]) and np.array_equal(regs[2], good[2])


def np_within(q, r):
    """Strictly inside the closed polygon r: on no edge (the same rounding as the device's test) and inside by the
    even-odd rule"""
    x, y = q[:, 0], q[:, 1]
    inside = np.zeros(len(q), bool)
    edge = np.zeros(len(q), bool)
    with np.errstate(divide="ignore", invalid="ignore"):
        for i in range(len(r)):
            a, b = r[i], r[i - 1]
            box = (x >= min(a[0], b[0])) & (x <= max(a[0], b[0])) & (y >= min(a[1], b[1])) & (y <= max(a[1], b[1]))
            edge |= box & ((b[0] - a[0]) * (y - a[1]) - (b[1] - a[1]) * (x - a[0]) == 0.)
            inside ^= ((a[1] > y) != (b[1] > y)) & (x < (b[0] - a[0]) * (y - a[1]) / (b[1] - a[1]) + a[0])
    return inside & ~edge


def _region_model(r):
    m = mrcal_b200.cameramodel(intrinsics=("LENSMODEL_OPENCV4", [500., 500., 320., 240., 0, 0, 0, 0]),
                               imagersize=(640, 480))
    m.valid_intrinsics_region(r)
    return m


def _regions_to_test():
    square = np.array([[10, 10], [50, 10], [50, 40], [10, 40]])
    concave = np.array([[5, 5], [45, 5], [45, 20], [20, 20], [20, 45], [5, 45]])
    mask = np.zeros((12, 12), bool)
    mask[1:5, 1:5] = True
    mask[5:9, 5:9] = True
    mask[1:5, 9:11] = True
    mask[4, 8] = True                                  # touches the first square's corner diagonally
    touching = np.array(regions.find_external_contours(mask)[0]) * 4
    th = np.linspace(0, 2 * np.pi, 5000, endpoint=False)
    circle = np.round(np.stack((2000 + 1500 * np.cos(th), 1100 + 1000 * np.sin(th)), -1))
    return dict(square=square, concave=concave, touching=touching, long=circle)


@pytest.mark.parametrize("name", ["square", "concave", "touching", "long"])
def test_is_within_region(name):
    r = _regions_to_test()[name]
    m = _region_model(r)
    rc = m.valid_intrinsics_region()
    lo, hi = rc.min(0) - 2, rc.max(0) + 2
    rng = np.random.default_rng(1)
    if name == "long":
        gx, gy = np.meshgrid(np.arange(lo[0], hi[0], 37.), np.arange(lo[1], hi[1], 23.))
        q = np.concatenate((np.stack((gx, gy), -1).reshape(-1, 2), rc, (rc + np.roll(rc, 1, 0)) / 2.,
                            rng.uniform(lo, hi, (4000, 2))))
    else:
        gx, gy = np.meshgrid(np.arange(lo[0], hi[0] + 1), np.arange(lo[1], hi[1] + 1))
        q = np.concatenate((np.stack((gx, gy), -1).reshape(-1, 2), (rc + np.roll(rc, 1, 0)) / 2.,
                            rng.uniform(lo, hi, (3000, 2)), np.arange(lo[0], hi[0], 0.25)[:, None] * (1, 0) + (0, 10)))
    q = np.concatenate((q, [[np.nan, 20.], [20., np.nan], [np.nan, np.nan]]))
    mask = mrcal_b200.is_within_valid_intrinsics_region(q, m)
    ref = np_within(q, rc)
    assert np.array_equal(mask, ref)
    assert ref.any() and (~ref).any()
    assert not mask[-3:].any()
    assert not mrcal_b200.is_within_valid_intrinsics_region(rc, m).any()       # the vertices are outside
    # the shape of q is kept
    assert mrcal_b200.is_within_valid_intrinsics_region(q[:12].reshape(3, 4, 2), m).shape == (3, 4)


def test_is_within_empty_and_none():
    m = _region_model(np.zeros((0, 2)))
    q = np.array([[1., 2.], [300., 200.], [np.nan, 0.]])
    assert mrcal_b200.is_within_valid_intrinsics_region(q, m).tolist() == [False] * 3
    m = mrcal_b200.cameramodel(intrinsics=("LENSMODEL_OPENCV4", [500., 500., 320., 240., 0, 0, 0, 0]),
                               imagersize=(640, 480))
    assert mrcal_b200.is_within_valid_intrinsics_region(q, m) is None


def test_region_drives_image_transformation_map(solved_opencv8):
    kw = solved_opencv8
    m = _models(kw)[1]
    s = np.std(mrcal_b200.measurements_board(kw).ravel())
    r = mrcal_b200._compute_valid_intrinsics_region(m, 2 * s, 0.5, 1.5 * s, 3, 0)
    assert r.shape[0] >= 4
    m.valid_intrinsics_region(r)
    mapxy = mrcal_b200.image_transformation_map(m, m, intrinsics_only=True, mask_valid_intrinsics_region_from=True)
    masked = (mapxy == -1).all(-1)
    W, H = m.imagersize()
    gx, gy = np.meshgrid(np.arange(0, W, 7.), np.arange(0, H, 7.))
    q = np.stack((gx, gy), -1).reshape(-1, 2)
    inside = mrcal_b200.is_within_valid_intrinsics_region(q, m)
    rc = m.valid_intrinsics_region()
    on_edge = np_within(q, rc) != inside                 # never: the strict tests agree
    assert not on_edge.any()
    near = np.zeros(len(q), bool)
    for i in range(len(rc)):                              # pixels within a pixel of an edge may go either way
        a, b = rc[i], rc[i - 1]
        d = b - a
        t = np.clip(((q - a) @ d) / max(d @ d, 1e-12), 0, 1)
        near |= np.linalg.norm(q - (a + t[:, None] * d), axis=-1) < 1.
    got = ~masked[::7, ::7].reshape(-1)
    assert inside.any() and (~inside).any()
    assert np.array_equal(got[~near], inside[~near])
