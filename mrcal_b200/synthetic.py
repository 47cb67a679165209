"""Synthetic calibration problems (host side, numpy only).

The reference builds its test/benchmark inputs with
mrcal.synthesize_board_observations() (mrcal/synthetic_data.py:236-554) and
test/test_calibration_helpers.py:calibration_baseline(); neither is importable
without numpysane. This module produces inputs with the same structure and the
same distribution of board poses (uniform noise of a given radius around a
nominal board-centre pose, keeping the frames every camera sees in full), for
the lens models the CUDA path supports. It is used by the tests, by
__graft_entry__.smoke() and by bench.py (BASELINE.json configs).

Nothing here is on the hot path: the projection below has no gradients and
exists only to manufacture observations.
"""
import numpy as np


# Not _poses_host's: bench.py loads this file by path, without the package, and this arithmetic fixes the benchmark's
# inputs bit for bit
def R_from_r(r):
    """Rodrigues vector(s) (...,3) -> rotation matrices (...,3,3)."""
    r = np.asarray(r, float)
    th = np.linalg.norm(r, axis=-1)[..., None, None]
    K = np.zeros(r.shape[:-1] + (3, 3))
    K[..., 0, 1], K[..., 0, 2] = -r[..., 2], r[..., 1]
    K[..., 1, 0], K[..., 1, 2] = r[..., 2], -r[..., 0]
    K[..., 2, 0], K[..., 2, 1] = -r[..., 1], r[..., 0]
    with np.errstate(invalid="ignore", divide="ignore"):
        b = np.where(th > 1e-8, np.sin(th) / th, 1. - th * th / 6.)
        c = np.where(th > 1e-8, (1. - np.cos(th)) / (th * th), 0.5 - th * th / 24.)
    return np.eye(3) + b * K + c * (K @ K)


def transform_rt(rt, p):
    """x -> R(r) x + t, broadcasting rt (...,6) against p (...,3)."""
    rt = np.asarray(rt, float)
    return np.einsum("...ij,...j->...i", R_from_r(rt[..., :3]), p) + rt[..., 3:]


def parse_splined(lensmodel):
    """'LENSMODEL_SPLINED_STEREOGRAPHIC_order=3_Nx=30_Ny=20_fov_x_deg=170' -> dict."""
    cfg = {}
    for tok in lensmodel[len("LENSMODEL_SPLINED_STEREOGRAPHIC_"):].replace("fov_x_deg", "fov").split("_"):
        k, v = tok.split("=")
        cfg[k] = int(v)
    margin = {2: 1, 3: 2}[cfg["order"]]
    u_edge = 2. * np.tan(cfg["fov"] / 2. * np.pi / 180. / 2.)
    cfg["segments_per_u"] = (cfg["Nx"] - 1 - margin) / (2. * u_edge)
    return cfg


def knots(lensmodel):
    c = parse_splined(lensmodel)
    ux = (np.arange(c["Nx"]) - (c["Nx"] - 1) / 2.) / c["segments_per_u"]
    uy = (np.arange(c["Ny"]) - (c["Ny"] - 1) / 2.) / c["segments_per_u"]
    return ux, uy


def _bspline_weights(order, t):
    t2 = t * t
    if order == 3:
        t3 = t2 * t
        return np.stack(((-t3 + 3 * t2 - 3 * t + 1) / 6., (3 * t3 / 2. - 3 * t2 + 2) / 3.,
                         (-3 * t3 + 3 * t2 + 3 * t + 1) / 6., t3 / 6.), axis=-1)
    return np.stack(((4 * t2 - 4 * t + 1) / 8., (3 - 4 * t2) / 4., (4 * t2 + 4 * t + 1) / 8.), axis=-1)


def project(p, lensmodel, intrinsics):
    """Pixel coordinates of camera-frame points p (...,3). No gradients."""
    p = np.asarray(p, float)
    intr = np.asarray(intrinsics, float)
    fxy, cxy = intr[0:2], intr[2:4]
    x, y, z = p[..., 0], p[..., 1], p[..., 2]
    if lensmodel == "LENSMODEL_PINHOLE":
        u = np.stack((x / z, y / z), -1)
    elif lensmodel.startswith("LENSMODEL_OPENCV"):
        k = np.zeros(12)
        k[:len(intr) - 4] = intr[4:]
        xn, yn = x / z, y / z
        r2 = xn * xn + yn * yn
        r4, r6 = r2 * r2, r2 * r2 * r2
        s = (1 + k[0] * r2 + k[1] * r4 + k[4] * r6) / (1 + k[5] * r2 + k[6] * r4 + k[7] * r6)
        u = np.stack((xn * s + 2 * k[2] * xn * yn + k[3] * (r2 + 2 * xn * xn) + k[8] * r2 + k[9] * r4,
                      yn * s + k[2] * (r2 + 2 * yn * yn) + 2 * k[3] * xn * yn + k[10] * r2 + k[11] * r4), -1)
    elif lensmodel == "LENSMODEL_CAHVOR":
        al, be, r0, r1, r2 = intr[4:9]
        o = np.array((np.sin(al) * np.cos(be), np.sin(be), np.cos(al) * np.cos(be)))
        w = p @ o
        tau = (p * p).sum(-1) / (w * w) - 1.
        mu = r0 + tau * r1 + tau * tau * r2
        pd = p + mu[..., None] * (p - w[..., None] * o)
        u = np.stack((pd[..., 0] / pd[..., 2], pd[..., 1] / pd[..., 2]), -1)
    elif lensmodel.startswith("LENSMODEL_CAHVORE_linearity="):
        # noncentral JPL model: theta by Newton's method, as the reference does it (cahvore.cc:77-116)
        lin = float(lensmodel[len("LENSMODEL_CAHVORE_linearity="):])
        al, be, r0, r1, r2, e0, e1, e2 = intr[4:12]
        o = np.array((np.sin(al) * np.cos(be), np.sin(be), np.cos(al) * np.cos(be)))
        zeta = p @ o
        ll = p - zeta[..., None] * o
        l = np.sqrt((ll * ll).sum(-1))
        th = np.arctan2(l, zeta)
        for _ in range(100):
            s_, c_ = np.sin(th), np.cos(th)
            E = e0 + e1 * th**2 + e2 * th**4
            ups = zeta * c_ + l * s_ + (c_ - 1.) * E - (th - s_) * (2. * e1 * th + 4. * e2 * th**3)
            step = (zeta * s_ - l * c_ - (th - s_) * E) / ups
            th = th - step
            if np.abs(step).max() < 1e-12:
                break
        chi = th if abs(lin) <= 1e-15 else (np.sin(th * lin) if lin < 0 else np.tan(th * lin)) / lin
        big = th > 1e-8
        chis = np.where(big, chi, 1.)
        pd = np.where(big[..., None], o * (l / chis)[..., None] + ll * (1. + r0 + r1 * chis**2 + r2 * chis**4)[..., None], p)
        u = np.stack((pd[..., 0] / pd[..., 2], pd[..., 1] / pd[..., 2]), -1)
    elif lensmodel == "LENSMODEL_LONLAT":
        u = np.stack((np.arctan2(x, z), np.arcsin(y / np.linalg.norm(p, axis=-1))), -1)
    elif lensmodel == "LENSMODEL_LATLON":
        u = np.stack((np.arcsin(x / np.linalg.norm(p, axis=-1)), np.arctan2(y, z)), -1)
    elif lensmodel == "LENSMODEL_STEREOGRAPHIC" or lensmodel.startswith("LENSMODEL_SPLINED_STEREOGRAPHIC"):
        scale = 2. / (np.linalg.norm(p, axis=-1) + z)
        u = np.stack((x * scale, y * scale), -1)
        if lensmodel != "LENSMODEL_STEREOGRAPHIC":
            c = parse_splined(lensmodel)
            Nx, Ny, order = c["Nx"], c["Ny"], c["order"]
            ctrl = intr[4:].reshape(Ny, Nx, 2)
            ix = u[..., 0] * c["segments_per_u"] + (Nx - 1) / 2.
            iy = u[..., 1] * c["segments_per_u"] + (Ny - 1) / 2.
            if order == 3:
                ix0 = np.clip(np.trunc(ix).astype(int), 1, Nx - 3)
                iy0 = np.clip(np.trunc(iy).astype(int), 1, Ny - 3)
            else:
                ix0 = np.clip(np.trunc(ix + 0.5).astype(int), 1, Nx - 2)
                iy0 = np.clip(np.trunc(iy + 0.5).astype(int), 1, Ny - 2)
            wx = _bspline_weights(order, ix - ix0)
            wy = _bspline_weights(order, iy - iy0)
            du = np.zeros(u.shape)
            for jy in range(order + 1):
                for jx in range(order + 1):
                    du += (wx[..., jx] * wy[..., jy])[..., None] * ctrl[iy0 - 1 + jy, ix0 - 1 + jx]
            u = u + du
    else:
        raise ValueError(f"synthetic.project(): unsupported lens model {lensmodel}")
    return u * fxy + cxy


def board_points(W, H, spacing, calobject_warp=None):
    """(H,W,3) board corners in the board frame, with the parabolic warp of
    mrcal.c:2794-2819 / ref_calibration_object() (mrcal/synthetic_data.py:25)."""
    xx, yy = np.meshgrid(np.arange(W, dtype=float), np.arange(H, dtype=float))
    pts = np.zeros((H, W, 3))
    pts[..., 0] = xx * spacing
    pts[..., 1] = yy * spacing
    if calobject_warp is not None:
        xr, yr = xx / (W - 1), yy / (H - 1)
        pts[..., 2] = calobject_warp[0] * 4. * xr * (1. - xr) + calobject_warp[1] * 4. * yr * (1. - yr)
    return pts


# camera geometry of the reference's 4-camera tests (test/test-basic-calibration.py:48-51),
# continued with the same ~1-2 m spacing for larger rigs
_RT_CAM_REF = np.array(((0., 0., 0., 0., 0., 0.),
                        (0.08, 0.2, 0.02, 1., 0.9, 0.1),
                        (0.01, 0.07, 0.2, 2.1, 0.4, 0.2),
                        (-0.1, 0.08, 0.08, 4.4, 0.2, 0.1),
                        (0.05, -0.1, 0.03, 5.6, 0.5, -0.1),
                        (-0.03, 0.12, -0.05, 6.9, 0.1, 0.15),
                        (0.02, -0.06, 0.1, 8.2, 0.6, 0.05),
                        (-0.07, 0.03, -0.02, 9.5, 0.3, -0.05)))

_CORE = np.array((1761.18, 1761.25, 1965.71, 1087.52))
_OPENCV_DIST = np.array((-0.0127, 0.0359, -0.00025, 0.00053, 0.0197, 0.0148, -0.0562, 0.05,
                         1e-4, -2e-4, 1.5e-4, -1e-4))


def true_intrinsics(lensmodel, Ncameras, rng):
    """A plausible truth: the reference's test cameras' core, per-camera jitter."""
    out = []
    for icam in range(Ncameras):
        core = _CORE * (1. + 0.01 * rng.uniform(-1, 1, 4))
        if lensmodel.startswith("LENSMODEL_SPLINED_STEREOGRAPHIC"):
            ux, uy = knots(lensmodel)
            UX, UY = np.meshgrid(ux, uy)
            # smooth, mostly-radial analytic field (SURVEY.md 8d), different per camera
            a = 1e-2 * (1. + 0.2 * icam)
            field = np.stack((a * (UX * UX - UY * UY) + 2e-3 * UX * (UX * UX + UY * UY),
                              a * (2. * UX * UY) + 2e-3 * UY * (UX * UX + UY * UY)), -1)
            out.append(np.concatenate((core, field.ravel())))
        elif lensmodel.startswith("LENSMODEL_OPENCV"):
            n = int(lensmodel[len("LENSMODEL_OPENCV"):])
            out.append(np.concatenate((core, _OPENCV_DIST[:n] * (1. + 0.1 * rng.uniform(-1, 1, n)))))
        elif lensmodel == "LENSMODEL_CAHVOR":
            out.append(np.concatenate((core, np.array((0.01, -0.02, 0.0, 0.03, 0.01)) * (1. + 0.1 * rng.uniform(-1, 1, 5)))))
        elif lensmodel.startswith("LENSMODEL_CAHVORE"):
            out.append(np.concatenate((core, np.array((0.01, -0.02, 0.0, 0.03, 0.01, 0.002, 0.01, -0.004)) * (1. + 0.1 * rng.uniform(-1, 1, 8)))))
        elif lensmodel in ("LENSMODEL_LONLAT", "LENSMODEL_LATLON"):
            out.append(core * np.array((1., 1., 1., 1.)))
        else:
            out.append(core)
    return np.array(out)


def synthesize_board_observations(lensmodel, intrinsics, rt_cam_ref_all, imagersize, W, H, spacing, calobject_warp,
                                  rt_ref_boardcenter, noiseradius, Nframes, rng, which="all"):
    """Random board poses that every ('all') or at least one ('some') camera sees in full.

    Returns q (Nframes,Ncameras,H,W,2), visible (Nframes,Ncameras) and
    rt_ref_frame (Nframes,6): the pose of the board frame (origin at corner 0,0)."""
    Ncam = len(intrinsics)
    center = np.array(((W - 1) * spacing / 2., (H - 1) * spacing / 2., 0.))
    pts = board_points(W, H, spacing, calobject_warp)
    qs, vis, rts = [], [], []
    n = 0
    while n < Nframes:
        chunk = max(64, 2 * (Nframes - n))
        rt_c = rt_ref_boardcenter + rng.uniform(-1., 1., (chunk, 6)) * noiseradius
        # board frame = boardcenter frame shifted by -center: same rotation
        R = R_from_r(rt_c[:, :3])
        rt_f = rt_c.copy()
        rt_f[:, 3:] = rt_c[:, 3:] - np.einsum("nij,j->ni", R, center)
        p_ref = np.einsum("nij,hwj->nhwi", R, pts) + rt_f[:, None, None, 3:]
        q = np.zeros((chunk, Ncam, H, W, 2))
        ok = np.zeros((chunk, Ncam), bool)
        for icam in range(Ncam):
            p_cam = transform_rt(rt_cam_ref_all[icam], p_ref)
            q[:, icam] = project(p_cam, lensmodel, intrinsics[icam])
            inview = (q[:, icam, ..., 0] >= 0) & (q[:, icam, ..., 1] >= 0) & \
                     (q[:, icam, ..., 0] <= imagersize[0] - 1) & (q[:, icam, ..., 1] <= imagersize[1] - 1) & \
                     (p_cam[..., 2] > 0.1)
            ok[:, icam] = inview.all(axis=(-1, -2))
        keep = ok.all(axis=1) if which == "all" else ok.any(axis=1)
        qs.append(q[keep]); vis.append(ok[keep]); rts.append(rt_f[keep])
        n += int(keep.sum())
    return np.concatenate(qs)[:Nframes], np.concatenate(vis)[:Nframes], np.concatenate(rts)[:Nframes]


def make_problem(lensmodel="LENSMODEL_OPENCV8", Ncameras=2, Nframes=20, W=10, H=10, spacing=0.1,
                 seed=0, pixel_noise=0.0, perturb=1.0, imagersize=(4000, 2200),
                 weights=(0.6, 1.0), which="all", Npoints=0, Npoints_fixed=0,
                 do_optimize_intrinsics_core=None, calobject_warp_true=(0.002, -0.005)):
    """An optimization_inputs dict (seed = perturbed truth) and the truth.

    Selections follow the reference's tests (test_calibration_helpers.py:363-370):
    everything optimised, the core locked for splined models, regularization on,
    outlier rejection off. All randomness comes from one default_rng(seed) stream
    in the order: intrinsics truth, board poses, weights, pixel noise, points,
    seed perturbations."""
    rng = np.random.default_rng(seed)
    splined = lensmodel.startswith("LENSMODEL_SPLINED_STEREOGRAPHIC")
    intr_true = true_intrinsics(lensmodel, Ncameras, rng)
    rt_cam_all = _RT_CAM_REF[:Ncameras].copy()
    if Ncameras > len(_RT_CAM_REF):
        raise ValueError(f"at most {len(_RT_CAM_REF)} cameras")
    warp_true = np.array(calobject_warp_true, float)
    x_center = -(Ncameras - 1) / 2. if Ncameras != 4 else -2.   # test-basic-calibration.py:68
    rt_center = np.array((0., 0., 0., x_center, 0., 4.0))
    radius = np.array((np.pi / 180. * 30., np.pi / 180. * 30., np.pi / 180. * 20., 2.5, 2.5, 2.0))
    if Ncameras >= 4:   # keep the acceptance rate of "every camera sees everything" workable
        rt_center[3] = -rt_cam_all[:, 3].mean() * 0.9
        rt_center[5] = 4.0 + 0.5 * (Ncameras - 4)
    q, vis, rt_frame_true = synthesize_board_observations(lensmodel, intr_true, rt_cam_all, imagersize, W, H, spacing,
                                                          warp_true, rt_center, radius, Nframes, rng, which)
    w = weights[0] + (weights[1] - weights[0]) * rng.uniform(0., 1., q.shape[:-1])
    if pixel_noise > 0:
        q = q + rng.normal(0., pixel_noise, q.shape) / w[..., None]
    idx, obs = [], []
    for iframe in range(Nframes):
        for icam in range(Ncameras):
            if vis[iframe, icam]:
                idx.append((iframe, icam, icam - 1))
                obs.append(np.concatenate((q[iframe, icam], w[iframe, icam][..., None]), -1))
    observations_board = np.ascontiguousarray(np.array(obs))
    indices = np.array(idx, np.int32)

    inputs = dict(lensmodel=lensmodel,
                  imagersizes=np.array([imagersize] * Ncameras, np.int32),
                  observations_board=observations_board,
                  indices_frame_camintrinsics_camextrinsics=indices,
                  calibration_object_spacing=spacing,
                  do_optimize_intrinsics_core=(not splined) if do_optimize_intrinsics_core is None
                  else do_optimize_intrinsics_core,
                  do_optimize_intrinsics_distortions=True,
                  do_optimize_extrinsics=Ncameras > 1,
                  do_optimize_frames=True,
                  do_optimize_calobject_warp=True,
                  do_apply_regularization=True,
                  do_apply_outlier_rejection=False)
    truth = dict(intrinsics=intr_true, rt_cam_ref=rt_cam_all[1:].copy(), rt_ref_frame=rt_frame_true,
                 calobject_warp=warp_true)

    if Npoints > 0:
        pts = np.stack((rng.uniform(-3., 3. + rt_cam_all[:, 3].max(), Npoints), rng.uniform(-3., 3., Npoints),
                        rng.uniform(3., 8., Npoints)), -1)
        io, oo = [], []
        for ip in range(Npoints):
            for icam in range(Ncameras):
                pc = transform_rt(rt_cam_all[icam], pts[ip])
                qq = project(pc, lensmodel, intr_true[icam])
                if pc[2] > 0.1 and 0 <= qq[0] <= imagersize[0] - 1 and 0 <= qq[1] <= imagersize[1] - 1:
                    io.append((ip, icam, icam - 1))
                    oo.append((qq[0], qq[1], 1.0))
        # a point seen by a single camera has a rank-2 (singular) 3x3 block: keep those seen at least twice.
        # And keep the reference's rule: point indices appear in order and cover all points
        nviews = np.bincount([i[0] for i in io], minlength=Npoints)
        keep = [k for k, i in enumerate(io) if nviews[i[0]] >= 2]
        io = [io[k] for k in keep]
        oo = [oo[k] for k in keep]
        seen = sorted(set(i[0] for i in io))
        remap = {old: new for new, old in enumerate(seen)}
        pts = pts[seen]
        io = [(remap[a], b, c) for a, b, c in io]
        order = np.argsort([i[0] for i in io], kind="stable")
        inputs["indices_point_camintrinsics_camextrinsics"] = np.array(io, np.int32)[order]
        oo = np.array(oo)[order]
        if pixel_noise > 0:
            oo[:, :2] += rng.normal(0., pixel_noise, oo[:, :2].shape)
        inputs["observations_point"] = np.ascontiguousarray(oo)
        inputs["Npoints_fixed"] = Npoints_fixed
        truth["points"] = pts

    # seed = truth perturbed (builder's choice, SURVEY.md 8d): distortions/knots
    # +N(0,1e-3*scale), poses +-(0.5 deg, 1 cm), warp 0
    s = perturb
    intr_seed = intr_true.copy()
    if splined:
        intr_seed[:, 4:] += s * 1e-3 * rng.normal(size=intr_seed[:, 4:].shape)
    else:
        intr_seed[:, :2] *= 1. + s * 2e-3 * rng.normal(size=(Ncameras, 2))
        intr_seed[:, 2:4] += s * 2.0 * rng.normal(size=(Ncameras, 2))
        intr_seed[:, 4:] += s * 1e-3 * rng.normal(size=intr_seed[:, 4:].shape)
    rt_cam_seed = truth["rt_cam_ref"].copy()
    rt_cam_seed[:, :3] += s * np.pi / 180. * 0.5 * rng.uniform(-1, 1, rt_cam_seed[:, :3].shape)
    rt_cam_seed[:, 3:] += s * 0.01 * rng.uniform(-1, 1, rt_cam_seed[:, 3:].shape)
    rt_frame_seed = rt_frame_true.copy()
    rt_frame_seed[:, :3] += s * np.pi / 180. * 0.5 * rng.uniform(-1, 1, rt_frame_seed[:, :3].shape)
    rt_frame_seed[:, 3:] += s * 0.01 * rng.uniform(-1, 1, rt_frame_seed[:, 3:].shape)
    inputs.update(intrinsics=np.ascontiguousarray(intr_seed),
                  rt_cam_ref=np.ascontiguousarray(rt_cam_seed),
                  rt_ref_frame=np.ascontiguousarray(rt_frame_seed),
                  calobject_warp=np.zeros(2))
    if Npoints > 0:
        inputs["points"] = np.ascontiguousarray(truth["points"] + s * 0.02 * rng.normal(size=truth["points"].shape))
    return inputs, truth


# BASELINE.json configs
def baseline_config(i, **overrides):
    splined = "LENSMODEL_SPLINED_STEREOGRAPHIC_order=3_Nx=30_Ny=20_fov_x_deg=170"
    cfg = {1: dict(lensmodel="LENSMODEL_OPENCV8", Ncameras=1, Nframes=30),
           2: dict(lensmodel="LENSMODEL_OPENCV8", Ncameras=2, Nframes=200),
           3: dict(lensmodel=splined, Ncameras=4, Nframes=400),
           4: dict(lensmodel=splined, Ncameras=4, Nframes=400),
           5: dict(lensmodel=splined, Ncameras=8, Nframes=1000, Npoints=2000)}[i]
    cfg.update(overrides)
    return make_problem(**cfg)
