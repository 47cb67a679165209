"""TEST INFRASTRUCTURE ONLY -- the reference's synthetic-data functions (mrcal/synthetic_data.py: ref_calibration_object,
synthesize_board_observations, make_perfect_observations; mrcal/utils.py: hypothesis_board_corner_positions)
restated in numpy, with every pose step and every projection made by the compiled reference (oracle/poseutils_ref.py,
oracle/ref.py), one element at a time. The random draws are the reference's, in its order, from the global np.random.

Also: the synthesis cases the tests run (cases()), the cameras they use (cameras()), and the decision margins
of each candidate frame, so that a test can assert that no decision lies within its tolerance of a threshold."""
import hashlib

import numpy as np

from oracle import poseutils_ref as PR
from oracle import ref

MODELS = ("LENSMODEL_PINHOLE", "LENSMODEL_STEREOGRAPHIC", "LENSMODEL_LONLAT", "LENSMODEL_LATLON",
          "LENSMODEL_OPENCV4", "LENSMODEL_OPENCV5", "LENSMODEL_OPENCV8", "LENSMODEL_OPENCV12", "LENSMODEL_CAHVOR",
          "LENSMODEL_CAHVORE_linearity=0.37", "LENSMODEL_CAHVORE_linearity=-0.25",
          "LENSMODEL_SPLINED_STEREOGRAPHIC_order=3_Nx=8_Ny=6_fov_x_deg=100",
          "LENSMODEL_SPLINED_STEREOGRAPHIC_order=2_Nx=8_Ny=6_fov_x_deg=100")   # test_project_gpu.MODELS
WHICH = ('all-cameras-must-see-full-board', 'some-cameras-must-see-full-board',
         'all-cameras-must-see-half-board', 'some-cameras-must-see-half-board')
IMAGERSIZE = (4000, 2200)


def ref_calibration_object(W, H, spacing, calobject_warp=None, x_corner0=0, x_corner1=None, Nx=None, y_corner0=0,
                           y_corner1=None, Ny=None):
    """(Ny,Nx,3); spacing: a scalar or (2,) of (x, y); calobject_warp: None or (2,). No broadcasting"""
    Nx = W if Nx is None else Nx
    Ny = H if Ny is None else Ny
    xs = np.linspace(x_corner0, W - 1 if x_corner1 is None else x_corner1, Nx)
    ys = np.linspace(y_corner0, H - 1 if y_corner1 is None else y_corner1, Ny)
    sx, sy = (spacing, spacing) if np.ndim(spacing) == 0 else spacing
    out = np.zeros((Ny, Nx, 3))
    out[..., 0] = xs[None, :] * sx
    out[..., 1] = ys[:, None] * sy
    if calobject_warp is not None:
        ux, uy = xs / (W - 1), ys / (H - 1)
        bx, by = 4. * ux * (1. - ux), 4. * uy * (1. - uy)
        # the two deflections added in turn, onto z = 0
        out[..., 2] = out[..., 2] + calobject_warp[0] * bx[None, :]
        out[..., 2] = out[..., 2] + calobject_warp[1] * by[:, None]
    return out


def _transform(Rt, p):
    """transform_point_Rt of the reference: Rt (N,4,3), p (N,3)"""
    return PR.transform_point_Rt(Rt, p, False)[0]


def _Rt(rt):
    return PR.Rt_from_rt(np.asarray(rt, np.float64).reshape(-1, 6), False)[0]


def rng_digest():
    """sha256 of np.random's whole state"""
    name, key, pos, has_gauss, cached = np.random.get_state()
    h = hashlib.sha256(key.tobytes())
    h.update(np.array((pos, has_gauss), np.int64).tobytes())
    h.update(np.float64(cached).tobytes())
    return h.hexdigest()


def synthesize_board_observations(cams, W, H, spacing, calobject_warp, rt_ref_boardcenter, noiseradius, Nframes,
                                  max_oblique_angle_deg=None, pcamera_nominal_ref=(0., 0., 0.),
                                  which='all-cameras-must-see-full-board'):
    """cams: [(lensmodel, intrinsics, rt_cam_ref, imagersize)]. Returns (q, Rt_ref_boardref, margins, Nchunks):
    margins (Ncandidates, 2) for every frame of every chunk, in draw order: the smallest distance of any corner's q
    from the image bounds over all cameras (inf if none is finite), and |costh - cos(max angle)| (inf without a
    maximum)"""
    Ncam, N = len(cams), W * H
    center = np.array(((W - 1) * spacing / 2., (H - 1) * spacing / 2., 0))
    board = (ref_calibration_object(W, H, spacing, calobject_warp) - center).reshape(-1, 3)
    Rt_cam_ref = [_Rt(c[2])[0] for c in cams]
    cosmax = None if max_oblique_angle_deg is None else np.cos(max_oblique_angle_deg * np.pi / 180.)
    q_all, Rt_all, margins, Nchunks = [], [], [], 0
    while True:
        Nchunks += 1
        rt = rt_ref_boardcenter + np.random.uniform(low=-1.0, high=1.0, size=(Nframes, 6)) * noiseradius
        Rt = _Rt(rt)
        # (Nframes*N,3): every corner of every frame, in the reference frame
        pref = _transform(np.repeat(Rt, N, axis=0), np.tile(board, (Nframes, 1)))
        q = np.zeros((Nframes, Ncam, N, 2))
        for c, (lm, intr, _, _) in enumerate(cams):
            pcam = _transform(np.repeat(Rt_cam_ref[c][None], Nframes * N, axis=0), pref)
            q[:, c] = ref.project(pcam, lm, intr).reshape(Nframes, N, 2)
        size = np.array([c[3] for c in cams], float)[None, :, None, :]
        inside = np.all((q >= 0) & (q <= size - 1), axis=-1)
        dist = np.minimum(np.abs(q), np.abs(size - 1 - q)).min(axis=-1)
        dist = np.where(np.isfinite(dist), dist, np.inf).reshape(Nframes, -1).min(axis=-1)
        keep = np.ones(Nframes, bool)
        dcos = np.full(Nframes, np.inf)
        if cosmax is not None:
            v = Rt[:, 3, :] - pcamera_nominal_ref
            v = v / np.sqrt(np.einsum('...i,...i', v, v))[:, None]
            costh = np.abs(np.einsum('...i,...i', v, Rt[:, :3, 2]))
            keep = costh > cosmax
            dcos = np.abs(costh - cosmax)
        margins.append(np.stack((dist, dcos), -1))
        nvis = inside.sum(axis=-1)
        full, half = nvis == N, nvis > N // 2
        sel = {WHICH[0]: full.all(-1), WHICH[1]: full.any(-1), WHICH[2]: half.all(-1), WHICH[3]: half.any(-1)}[which]
        keep &= sel
        q_all.append(q[keep])
        Rt_all.append(Rt[keep])
        if sum(len(a) for a in q_all) >= Nframes:
            break
    q = np.concatenate(q_all)[:Nframes].reshape(Nframes, Ncam, H, W, 2)
    Rt = np.concatenate(Rt_all)[:Nframes]
    shift = np.concatenate((np.eye(3), -center[None]))
    Rt = PR.compose_Rt(Rt, np.repeat(shift[None], len(Rt), axis=0))[0] if len(Rt) else Rt
    return q, Rt, np.concatenate(margins), Nchunks


def cameras(lensmodels, seed):
    """[(lensmodel, intrinsics, rt_cam_ref, imagersize)]: cameras 0.4 m apart along x, slightly rotated, all looking
    along +z"""
    from mrcal_b200 import synthetic
    rng = np.random.default_rng(seed)
    out = []
    for c, lm in enumerate(lensmodels):
        intr = synthetic.true_intrinsics(lm, 1, rng)[0]
        rt = np.array((0.02 * c, -0.01 * c, 0.015 * c, -0.4 * c, 0.05 * c, 0.))
        out.append((lm, intr, rt, IMAGERSIZE))
    return out


def cases():
    """[(key, kwargs)]: the synthesis cases. Every lens model of MODELS with 1 to 4 cameras, every `which`, with and
    without warp and an oblique-angle limit; one case mixing three lens models; one that needs several chunks"""
    out = []
    for i, lm in enumerate(MODELS):
        Ncam = 1 + i % 4
        out.append((f"{i:02d}_{lm}", dict(lensmodels=[lm] * Ncam, seed=100 + i, W=5, H=4, spacing=0.08,
                                          calobject_warp=None if i % 2 else np.array((0.002, -0.005)),
                                          rt_ref_boardcenter=np.array((0., 0., 0., -0.2 * (Ncam - 1), 0., 3.)),
                                          noiseradius=np.array((0.35, 0.35, 0.3, 2.5, 1.6, 0.8)),
                                          Nframes=7, max_oblique_angle_deg=None if i % 3 else 35.,
                                          which=WHICH[i % 4])))
    mixed = ["LENSMODEL_OPENCV8", "LENSMODEL_SPLINED_STEREOGRAPHIC_order=3_Nx=8_Ny=6_fov_x_deg=100",
             "LENSMODEL_CAHVORE_linearity=0.37"]
    out.append(("mixed", dict(lensmodels=mixed, seed=200, W=6, H=5, spacing=0.06, calobject_warp=np.array((0.003, 0.001)),
                              rt_ref_boardcenter=np.array((0., 0., 0., -0.4, 0., 2.5)),
                              noiseradius=np.array((0.3, 0.3, 0.3, 0.8, 0.5, 0.4)), Nframes=6,
                              max_oblique_angle_deg=50., which=WHICH[0])))
    out.append(("chunks", dict(lensmodels=["LENSMODEL_OPENCV4"] * 2, seed=201, W=4, H=3, spacing=0.1,
                               calobject_warp=None, rt_ref_boardcenter=np.array((0., 0., 0., -0.2, 0., 3.)),
                               noiseradius=np.array((0.4, 0.4, 0.4, 4.5, 3.0, 1.0)), Nframes=5,
                               max_oblique_angle_deg=40., which=WHICH[0])))
    return out


def run_case(kw):
    """(q, Rt_ref_boardref, margins, Nchunks, rng digest) of one case, from np.random.seed(kw['seed'])"""
    np.random.seed(kw["seed"])
    cams = cameras(kw["lensmodels"], kw["seed"])
    q, Rt, margins, Nchunks = synthesize_board_observations(
        cams, kw["W"], kw["H"], kw["spacing"], kw["calobject_warp"], kw["rt_ref_boardcenter"], kw["noiseradius"],
        kw["Nframes"], max_oblique_angle_deg=kw["max_oblique_angle_deg"], which=kw["which"])
    return q, Rt, margins, Nchunks, rng_digest()


def hypothesis_board_corner_positions(icam_intrinsics=None, idx_inliers=None, **inputs):
    """The reference's four arrays"""
    obs = inputs["observations_board"]
    idx = inputs["indices_frame_camintrinsics_camextrinsics"]
    Nobs, H, W = obs.shape[:3]
    board = ref_calibration_object(W, H, inputs["calibration_object_spacing"], inputs.get("calobject_warp"))
    Rt_ref_frame = _Rt(inputs["rt_ref_frame"])[idx[:, 0]]
    rt_cam = inputs.get("rt_cam_ref")
    Rt_cams = np.concatenate((np.concatenate((np.eye(3), np.zeros((1, 3))))[None],
                              _Rt(rt_cam) if rt_cam is not None and len(rt_cam) else np.zeros((0, 4, 3))))
    Rt_cam_frame = PR.compose_Rt(Rt_cams[idx[:, 2] + 1], Rt_ref_frame)[0]
    pcam = _transform(np.repeat(Rt_cam_frame, H * W, axis=0), np.tile(board.reshape(-1, 3), (Nobs, 1)))
    pcam = pcam.reshape(Nobs, H, W, 3)
    inl = obs[..., 2] > 0 if idx_inliers is None else idx_inliers.copy()
    outl = ~inl
    if icam_intrinsics is None:
        return pcam, pcam, pcam[inl], pcam[outl]
    mine = idx[:, 1] == icam_intrinsics
    inl[~mine] = False
    outl[~mine] = False
    return pcam, pcam[mine], pcam[inl], pcam[outl]


def perfect_projections(inputs):
    """(q_board (Nobs,H,W,2) or None, q_point (Nobs_point,2) or None): the perfect observations"""
    lm, intr = inputs["lensmodel"], inputs["intrinsics"]
    q_board = q_point = None
    idx = inputs.get("indices_frame_camintrinsics_camextrinsics")
    if idx is not None and idx.size:
        pcam = hypothesis_board_corner_positions(**inputs)[0]
        q_board = np.zeros(pcam.shape[:-1] + (2,))
        for c in np.unique(idx[:, 1]):
            s = idx[:, 1] == c
            q_board[s] = ref.project(pcam[s].reshape(-1, 3), lm, intr[c]).reshape(q_board[s].shape)
    idx = inputs.get("indices_point_camintrinsics_camextrinsics")
    if idx is not None and idx.size:
        rt_cam = inputs.get("rt_cam_ref")
        Rt_cams = np.concatenate((np.concatenate((np.eye(3), np.zeros((1, 3))))[None],
                                  _Rt(rt_cam) if rt_cam is not None and len(rt_cam) else np.zeros((0, 4, 3))))
        pcam = _transform(Rt_cams[idx[:, 2] + 1], inputs["points"][idx[:, 0]])
        q_point = np.zeros((len(idx), 2))
        for c in np.unique(idx[:, 1]):
            s = idx[:, 1] == c
            q_point[s] = ref.project(pcam[s], lm, intr[c])
    return q_board, q_point


def make_perfect_observations(inputs, observed_pixel_uncertainty):
    """The reference's function with a given sigma, in place"""
    q_board, q_point = perfect_projections(inputs)
    if q_board is not None:
        inputs["observations_board"][..., :2] = q_board
    if q_point is not None:
        inputs["observations_point"][..., :2] = q_point
    if observed_pixel_uncertainty == 0:
        return
    add_noise(inputs, observed_pixel_uncertainty)


def add_noise(inputs, observed_pixel_uncertainty):
    """The reference's noise step, in place: boards first, then points; weights <= 0 set to 1 through a view"""
    for what in ("observations_board", "observations_point"):
        obs = inputs.get(what)
        if obs is not None and obs.size:
            noise = observed_pixel_uncertainty * np.random.randn(*obs[..., :2].shape)
            w = obs[..., 2:3]   # a view
            w[w <= 0] = 1.
            obs[..., :2] += noise / w
