"""Image reprojection on the device: transform_image() against OpenCV's results and the numpy restatement of its
rule, its torch path against its numpy path, image_transformation_map() against an independent composition of
unproject/transform/project (and the compiled reference's, where it is built), against OpenCV's
initUndistortRectifyMap(), its mask against a numpy crossing-number rule, the reference's test-pylib-projections.py,
and determinism."""
import os

import numpy as np
import pytest

import mrcal_b200
from mrcal_b200._poses_host import rt_from_Rt

import remap_np

pytestmark = pytest.mark.gpu

MODELS = os.path.join(os.path.dirname(__file__), "golden", "cameramodels")
FIXTURE = os.path.join(os.path.dirname(__file__), "golden", "transform_image.npz")
DTYPES = {"uint8": np.uint8, "uint16": np.uint16, "float32": np.float32}


def _model(name):
    return mrcal_b200.cameramodel(os.path.join(MODELS, name))


####################################################################################################
# transform_image()
####################################################################################################
def _fixture_keys(f):
    return sorted({k[:-len("_result")] for k in f.files if k.endswith("_result") and k.split("_")[0] in DTYPES})


def test_transform_image_matches_opencv_and_the_rule():
    f = np.load(FIXTURE)
    keys = _fixture_keys(f)
    assert len(keys) == 24
    for key in keys:
        p = key + "_"
        interpolation = int(key.split("_i")[-1].split("_")[0])
        border = int(key.split("_b")[-1])
        image, mapxy = f[p + "image"], f[p + "mapxy"]
        out = f[p + "out"].copy()
        r = mrcal_b200.transform_image(image, mapxy, out=out, borderMode=border, borderValue=tuple(f[p + "border_value"]),
                                       interpolation=interpolation)
        assert r is out
        remap_np.assert_matches_opencv(r, f[p + "result"], image, mapxy,
                                       key.startswith("float32") and interpolation == 1 and border == 5)
        rule = remap_np.remap(image, mapxy, out=f[p + "out"], border=border, border_value=f[p + "border_value"],
                              interpolation=interpolation)
        np.testing.assert_array_equal(r, rule, err_msg=key)


@pytest.mark.parametrize("dtype", [np.uint8, np.uint16, np.float32])
@pytest.mark.parametrize("channels", [1, 3])
def test_transform_image_defaults_and_strided_rows(dtype, channels):
    big = remap_np.seeded_image(61, 83, channels, dtype, 5)
    image = big[7:50, 11:70]                      # rows strided: a crop of a larger image
    mapxy = remap_np.special_map(37, 53, 43, 59, 6)
    r = mrcal_b200.transform_image(image, mapxy, borderValue=9)
    np.testing.assert_array_equal(r, remap_np.remap(np.ascontiguousarray(image), mapxy, border=0, border_value=9,
                                                    interpolation=1))
    # transparent without out: untouched pixels are 0
    r = mrcal_b200.transform_image(image, mapxy, borderMode=mrcal_b200.BORDER_TRANSPARENT,
                                   interpolation=mrcal_b200.INTER_NEAREST)
    np.testing.assert_array_equal(r, remap_np.remap(np.ascontiguousarray(image), mapxy, border=5, interpolation=0))
    r2 = mrcal_b200.transform_image(image, mapxy, borderMode=mrcal_b200.BORDER_TRANSPARENT,
                                    interpolation=mrcal_b200.INTER_NEAREST)
    assert r.tobytes() == r2.tobytes()


def test_transform_image_torch_path_is_the_numpy_path():
    torch = pytest.importorskip("torch")
    f = np.load(FIXTURE)
    stream = torch.cuda.Stream()
    for key in _fixture_keys(f):
        p = key + "_"
        interpolation = int(key.split("_i")[-1].split("_")[0])
        border = int(key.split("_b")[-1])
        kw = dict(borderMode=border, borderValue=tuple(f[p + "border_value"]), interpolation=interpolation)
        ref = mrcal_b200.transform_image(f[p + "image"], f[p + "mapxy"], out=f[p + "out"].copy(), **kw)
        image = torch.from_numpy(f[p + "image"].copy()).cuda()
        mapxy = torch.from_numpy(f[p + "mapxy"].copy()).cuda()
        with torch.cuda.stream(stream):
            out = torch.from_numpy(f[p + "out"].copy()).cuda()
            r = mrcal_b200.transform_image(image, mapxy, out=out, **kw)
            r_new = mrcal_b200.transform_image(image, mapxy, **kw) if border == 0 else None
        stream.synchronize()
        assert r is out and r.is_cuda
        assert r.cpu().numpy().tobytes() == ref.tobytes(), key
        if r_new is not None:
            assert r_new.cpu().numpy().tobytes() == ref.tobytes(), key
    # on the default stream too
    image = torch.from_numpy(f["uint8_c3_i1_b0_image"].copy()).cuda()
    mapxy = torch.from_numpy(f["uint8_c3_i1_b0_mapxy"].copy()).cuda()
    r = mrcal_b200.transform_image(image, mapxy)
    ref = mrcal_b200.transform_image(image.cpu().numpy(), mapxy.cpu().numpy())
    assert r.cpu().numpy().tobytes() == ref.tobytes()
    # a contiguous map whose data starts an odd number of floats into its storage: only 4-byte aligned
    buf = torch.empty(mapxy.numel() + 1, dtype=torch.float32, device=mapxy.device)
    view = buf[1:].view(mapxy.shape)
    view.copy_(mapxy)
    assert view.is_contiguous() and view.data_ptr() % 8 == 4
    r = mrcal_b200.transform_image(image, view)
    assert r.cpu().numpy().tobytes() == ref.tobytes()


def test_transform_image_device_refuses_misaligned_buffers():
    """The C entry point of the device path refuses element-misaligned buffers before any launch"""
    import ctypes as C
    from mrcal_b200 import _capi
    torch = pytest.importorskip("torch")
    image = torch.zeros(2 * 8 * 8 + 1, dtype=torch.uint16, device="cuda")
    mapxy = torch.zeros((4, 4, 2), dtype=torch.float32, device="cuda")
    out = torch.zeros((4, 4), dtype=torch.uint16, device="cuda")
    bv = (C.c_double * 3)(0., 0., 0.)
    for img_ptr, stride, map_ptr in ((image.data_ptr() + 1, 16, mapxy.data_ptr()),
                                     (image.data_ptr(), 15 + 2, mapxy.data_ptr()),
                                     (image.data_ptr(), 16, mapxy.data_ptr() + 2)):
        assert not _capi.lib.mrcal_b200_transform_image_device(out.data_ptr(), img_ptr, 8, 8, stride, 1, 1, map_ptr,
                                                               4, 4, 1, 0, bv, None)
        assert "must be aligned" in _capi.last_error()
    torch.cuda.synchronize()


def test_transform_image_full_resolution_rectification():
    """A 4000x2200 RGB image through a rectification map of rectification_maps(): bit-exact to the rule"""
    models = [_model("cam0.opencv8.cameramodel"), _model("cam1.opencv8.cameramodel")]
    models_rectified = mrcal_b200.rectified_system(models, az_fov_deg=90., el_fov_deg=50.)
    maps = mrcal_b200.rectification_maps(models, models_rectified)
    W, H = models[0].imagersize()
    image = remap_np.seeded_image(int(H), int(W), 3, np.uint8, 11)
    for i in range(2):
        r = mrcal_b200.transform_image(image, maps[i])
        np.testing.assert_array_equal(r, remap_np.remap(image, maps[i]))


####################################################################################################
# image_transformation_map()
####################################################################################################
def _shrunk(m, k=0.1):
    """model m with its imager and core scaled by k: the same lens, fewer pixels"""
    lensmodel, intr = m.intrinsics()
    intr = intr.copy()
    intr[:4] *= k
    W, H = m.imagersize()
    return mrcal_b200.cameramodel(intrinsics=(lensmodel, intr), imagersize=(round(W * k), round(H * k)),
                                  rt_cam_ref=m.rt_cam_ref())


def _models():
    return {
        "opencv8": _shrunk(_model("cam0.opencv8.cameramodel")),
        "splined": _shrunk(_model("cam0.splined.cameramodel")),
        "cahvor": mrcal_b200.cameramodel(intrinsics=("LENSMODEL_CAHVOR", np.array((380., 385., 199., 111., 0.02, -0.01,
                                                                                    0., -0.05, 0.01))),
                                         imagersize=(400, 220)),
        "latlon": mrcal_b200.cameramodel(intrinsics=("LENSMODEL_LATLON", np.array((250., 250., 200., 110.))),
                                         imagersize=(400, 220)),
        "pinhole": mrcal_b200.cameramodel(intrinsics=("LENSMODEL_PINHOLE", np.array((300., 300., 200., 110.))),
                                          imagersize=(400, 220)),
    }


PAIRS = [("opencv8", "pinhole"), ("splined", "pinhole"), ("pinhole", "opencv8"), ("cahvor", "latlon"),
         ("latlon", "splined"), ("opencv8", "cahvor"), ("pinhole", "pinhole"), ("splined", "opencv8")]
MODES = {"infinity": {}, "distance": dict(distance=10.), "plane": dict(plane_n=np.array((0.1, 0.2, 1.)), plane_d=20.),
         "intrinsics_only": dict(intrinsics_only=True)}


def _posed(models, name_from, name_to):
    m_from = mrcal_b200.cameramodel(models[name_from])
    m_to = mrcal_b200.cameramodel(models[name_to])
    m_from.rt_cam_ref(np.array((0.01, -0.02, 0.005, 0.3, -0.1, 0.05)))
    m_to.rt_cam_ref(np.array((-0.015, 0.01, 0.02, -0.2, 0.05, 0.1)))
    return m_from, m_to


def _compose(m_from, m_to, mode, unproject, project, step=1):
    """unproject -> the reference's transformation in numpy -> project, in fp64, on every step-th row and column of
    model_to's pixels"""
    W, H = m_to.imagersize()
    grid = np.ascontiguousarray(np.stack(np.meshgrid(np.arange(0, W, step), np.arange(0, H, step)), axis=-1),
                                dtype=float)
    v = unproject(grid, *m_to.intrinsics())
    A, B = m_to.Rt_cam_ref(), m_from.Rt_ref_cam()
    Rt = np.vstack((A[:3] @ B[:3], A[:3] @ B[3] + A[3]))
    R, t = Rt[:3], Rt[3]
    kw = MODES[mode]
    if mode == "plane":
        A_to_from = kw["plane_d"] * R + np.outer(t, kw["plane_n"])
        v = v @ np.linalg.inv(A_to_from).T
    elif mode == "distance":
        p = v / np.linalg.norm(v, axis=-1)[..., None] * kw["distance"]
        v = p @ R - R.T @ t
    elif mode == "infinity":
        v = v @ R
    return project(v, *m_from.intrinsics())


def _assert_within_one_ulp(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    assert np.array_equal(np.isnan(a), np.isnan(b))
    ok = ~np.isnan(a)
    d = np.abs(a[ok].astype(np.float64) - b[ok])
    assert np.all(d <= np.spacing(np.maximum(np.abs(a[ok]), np.abs(b[ok])))), d.max()


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("pair", PAIRS, ids=["-".join(p) for p in PAIRS])
def test_image_transformation_map_against_composition(pair, mode):
    models = _models()
    m_from, m_to = _posed(models, *pair)
    mapxy = mrcal_b200.image_transformation_map(m_from, m_to, **MODES[mode])
    W, H = m_to.imagersize()
    assert mapxy.shape == (H, W, 2) and mapxy.dtype == np.float32
    q = _compose(m_from, m_to, mode, mrcal_b200.unproject, mrcal_b200.project)
    _assert_within_one_ulp(mapxy, q)
    assert np.isfinite(mapxy).mean() > 0.5
    again = mrcal_b200.image_transformation_map(m_from, m_to, **MODES[mode])
    assert mapxy.tobytes() == again.tobytes()


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("pair", [("opencv8", "pinhole"), ("opencv8", "latlon"), ("latlon", "pinhole")],
                         ids=["opencv8-pinhole", "opencv8-latlon", "latlon-pinhole"])
def test_image_transformation_map_against_compiled_reference(pair, mode):
    from oracle import ref
    if not ref.available():
        pytest.skip("oracle/_ref not built")
    models = _models()
    m_from, m_to = _posed(models, *pair)
    mapxy = mrcal_b200.image_transformation_map(m_from, m_to, **MODES[mode])
    q = _compose(m_from, m_to, mode, lambda q, lm, i: ref.unproject(q, lm, i).reshape(q.shape[:-1] + (3,)),
                 lambda v, lm, i: ref.project(v, lm, i).reshape(v.shape[:-1] + (2,)))
    both = np.isfinite(q).all(-1) & np.isfinite(mapxy).all(-1)
    assert both.mean() > 0.99
    assert np.abs(mapxy[both] - q[both]).max() <= 1e-6 + np.spacing(np.float32(np.abs(q[both]).max()))


ITERATIVE_TO = [("pinhole", "splined"), ("cahvor", "opencv8"), ("splined", "cahvor")]


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("pair", ITERATIVE_TO, ids=["-".join(p) for p in ITERATIVE_TO])
def test_image_transformation_map_iterative_against_compiled_reference(pair, mode):
    """model_to without a closed-form unprojection. The oracle solves it on the host, point by point, so every 5th
    row and column is compared; where the oracle's solve did not converge (its ray does not reproject to its pixel)
    there is nothing to compare"""
    from oracle import ref
    if not ref.available():
        pytest.skip("oracle/_ref not built")
    step = 5
    models = _models()
    m_from, m_to = _posed(models, *pair)
    mapxy = mrcal_b200.image_transformation_map(m_from, m_to, **MODES[mode])[::step, ::step]
    lm_to, intr_to = m_to.intrinsics()
    W, H = m_to.imagersize()
    grid = np.stack(np.meshgrid(np.arange(0, W, step), np.arange(0, H, step)), axis=-1).astype(float)
    converged = np.abs(ref.project(ref.unproject(grid, lm_to, intr_to), lm_to, intr_to).reshape(grid.shape) -
                       grid).max(-1) < 1e-6
    q = _compose(m_from, m_to, mode, lambda q, lm, i: ref.unproject(q, lm, i).reshape(q.shape[:-1] + (3,)),
                 lambda v, lm, i: ref.project(v, lm, i).reshape(v.shape[:-1] + (2,)), step=step)
    both = converged & np.isfinite(q).all(-1) & np.isfinite(mapxy).all(-1)
    assert both.mean() > 0.9
    assert np.abs(mapxy[both] - q[both]).max() <= 1e-6 + np.spacing(np.float32(np.abs(q[both]).max()))


def test_image_transformation_map_against_opencv_undistortion():
    """The general path for OPENCV8 -> pinhole, which the reference hands to cv2.initUndistortRectifyMap()"""
    f = np.load(FIXTURE)
    m = _model("cam0.opencv8.cameramodel")
    m.rt_cam_ref(np.zeros(6))
    worst = {}
    for key in ("undistort_", "rotated_"):
        pinhole = mrcal_b200.pinhole_model_for_reprojection(m, scale_focal=1., scale_image=0.1)
        pinhole.rt_cam_ref(rt_from_Rt(np.vstack((f[key + "R_to_from"], np.zeros(3)))))
        mapxy = mrcal_b200.image_transformation_map(m, pinhole)[::4, ::4]
        ref = f[key + "mapxy"]
        assert mapxy.shape == ref.shape
        # wherever the ray is in front of model_from
        W, H = pinhole.imagersize()
        grid = np.stack(np.meshgrid(np.arange(W), np.arange(H)), axis=-1)[::4, ::4].astype(float)
        v = mrcal_b200.unproject(grid, *pinhole.intrinsics()) @ f[key + "R_to_from"]
        front = v[..., 2] > 0
        worst[key] = np.abs(mapxy[front] - ref[front]).max()
    # measured on an H100: bit-identical at every sampled pixel
    assert max(worst.values()) == 0., worst


def _segment_distance(q, a, b):
    ab = b - a
    s = np.clip(((q - a) @ ab) / (ab @ ab), 0., 1.)
    return np.linalg.norm(q - (a + s[..., None] * ab), axis=-1)


def _crossing_number(q, P):
    c = np.zeros(q.shape[:-1], bool)
    x, y = q[..., 0], q[..., 1]
    for i in range(len(P)):
        j = i - 1
        with np.errstate(invalid="ignore", divide="ignore"):
            cross = ((P[i, 1] > y) != (P[j, 1] > y)) & \
                (x < (P[j, 0] - P[i, 0]) * (y - P[i, 1]) / (P[j, 1] - P[i, 1]) + P[i, 0])
        c ^= cross
    return c


@pytest.mark.parametrize("shape", ["convex", "concave"])
def test_mask_valid_intrinsics_region(shape):
    models = _models()
    m_from, m_to = _posed(models, "opencv8", "pinhole")
    W, H = m_from.imagersize()
    if shape == "convex":
        th = np.linspace(0, 2 * np.pi, 13)
        P = np.stack((W / 2 + 0.4 * W * np.cos(th), H / 2 + 0.4 * H * np.sin(th)), axis=-1)
    else:
        # a star: 7 points, closed
        th = np.linspace(0, 2 * np.pi, 15)
        r = np.where(np.arange(15) % 2 == 0, 0.45, 0.2)
        P = np.stack((W / 2 + r * W * np.cos(th), H / 2 + r * H * np.sin(th)), axis=-1)
    P[-1] = P[0]
    m_from = mrcal_b200.cameramodel(intrinsics=m_from.intrinsics(), imagersize=m_from.imagersize(),
                                    rt_cam_ref=m_from.rt_cam_ref(), valid_intrinsics_region=P)
    masked = mrcal_b200.image_transformation_map(m_from, m_to, mask_valid_intrinsics_region_from=True)
    plain = mrcal_b200.image_transformation_map(m_from, m_to)
    q = _compose(m_from, m_to, "infinity", mrcal_b200.unproject, mrcal_b200.project)
    inside = _crossing_number(q, P)
    near = np.zeros(inside.shape, bool)
    for i in range(1, len(P)):
        near |= _segment_distance(q, P[i - 1], P[i]) < 1e-9
    keep = ~near
    assert inside[keep].any() and (~inside[keep]).any()
    expected = np.where(inside[..., None], plain, np.float32(-1.))
    np.testing.assert_array_equal(masked[keep], expected[keep])
    # a NaN point is outside
    assert np.all(masked[np.isnan(plain).any(-1)] == -1.)
    assert masked.tobytes() == mrcal_b200.image_transformation_map(m_from, m_to,
                                                                   mask_valid_intrinsics_region_from=True).tobytes()


####################################################################################################
# the reference's test/test-pylib-projections.py
####################################################################################################
def _fit_check(scale_focal, intrinsics, v, W, H, eps=1e-2):
    """all projections inside the imager, at least one on its edge"""
    intrinsics = intrinsics.copy()
    intrinsics[:2] *= scale_focal
    q = mrcal_b200.project(v, "LENSMODEL_PINHOLE", intrinsics)
    if any(q[:, 0] < -eps) or any(q[:, 0] > W - 1 + eps) or any(q[:, 1] < -eps) or any(q[:, 1] > H - 1 + eps):
        return ": Some points lie out of bounds"
    on_edge = (np.abs(q[:, 0]) < eps) | (np.abs(q[:, 0] - (W - 1)) < eps) | (np.abs(q[:, 1]) < eps) | \
        (np.abs(q[:, 1] - (H - 1)) < eps)
    return "" if any(on_edge) else ": No points lie on the edge"


def test_pylib_projections():
    m = _model("cam0.opencv8.cameramodel")
    W, H = m.imagersize()
    core = m.intrinsics()[1][:4]
    assert mrcal_b200.scale_focal__best_pinhole_fit(m, None) == 1.0
    cases = [("corners", ((0, 0), (W - 1, 0), (0, H - 1), (W - 1, H - 1))),
             ("centers-horizontal", ((0, (H - 1.) / 2.), (W - 1, (H - 1.) / 2.))),
             ("centers-vertical", (((W - 1.) / 2., 0.), ((W - 1.) / 2., H - 1.)))]
    cases.append((np.array(cases[2][1], dtype=float), cases[2][1]))
    for fit, q in cases:
        v = mrcal_b200.unproject(np.array(q, dtype=float), *m.intrinsics())
        assert _fit_check(mrcal_b200.scale_focal__best_pinhole_fit(m, fit), core, v, W, H) == ""
    # pinhole_model_for_reprojection() applies that scale
    p = mrcal_b200.pinhole_model_for_reprojection(m, "corners")
    np.testing.assert_allclose(p.intrinsics()[1][:2], core[:2] * mrcal_b200.scale_focal__best_pinhole_fit(m, "corners"),
                               rtol=1e-15)
