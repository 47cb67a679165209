"""Geometric seeding of a calibration solve (host side, numpy only).

The step BEFORE the hot path: from chessboard observations alone, estimate the
camera poses and the pose of the board in every frame, assuming a stereographic
lens with a guessed focal length. What comes out is the seed that
mrcal-calibrate-cameras hands to the first optimize() call
(mrcal-calibrate-cameras:386-423). Mirrors, with the same names, arguments and
return conventions:

    seed_stereographic()                          mrcal/calibration.py:1398-1608
    estimate_monocular_calobject_poses_Rt_tocam() mrcal/calibration.py:622-781
    estimate_joint_frame_poses()                  mrcal/calibration.py:1186-1396
    (_estimate_camera_poses                       mrcal/calibration.py:925-1101,
     mrcal_traverse_sensor_links                  traverse-sensor-links.c,
     align_procrustes_points_Rt01                 poseutils.c / mrcal/poseutils.py)

The reference solves the per-observation pose problem with OpenCV's solvePnP();
OpenCV is not a dependency here, so the same problem (a planar target seen
through an ideal pinhole) is solved directly: homography by DLT, pose from the
homography, then a few Gauss-Newton steps on the pinhole reprojection error --
which is what solvePnP's iterative method does for a planar target. These are
seeds: the reference's own tests pin them only through the quality of the final
calibration (test/test-basic-calibration.py).

Nothing here runs on the GPU and nothing here is on the hot path.
"""
import heapq

import numpy as np

# absolute, so that this file also runs when loaded by its path rather than as part of the package
from mrcal_b200._poses_host import R_from_r, Rt_from_rt, compose_Rt, invert_Rt, r_from_R, rt_from_Rt, transform_point_Rt
from mrcal_b200.synthetic_data import ref_calibration_object


def align_procrustes_points_Rt01(p0, p1):
    """The rigid transform Rt01 with p0 ~ Rt01(p1), least squares (Kabsch). p0, p1: (N,3)."""
    p0 = np.asarray(p0, float).reshape(-1, 3)
    p1 = np.asarray(p1, float).reshape(-1, 3)
    if p0.shape[0] < 3:
        raise RuntimeError("align_procrustes_points_Rt01(): need at least 3 points")
    c0, c1 = p0.mean(0), p1.mean(0)
    M = (p0 - c0).T @ (p1 - c1)
    U, S, Vt = np.linalg.svd(M)
    d = np.sign(np.linalg.det(U @ Vt))
    R = U @ np.diag((1., 1., d)) @ Vt
    return np.concatenate((R, (c0 - R @ c1)[None]), 0)


# --------------------------------------------------------------------------- lens models needed for seeding
def _unproject_stereographic(q, fxycxy):
    """mrcal_unproject_stereographic (mrcal.c:1560-1620): pixel -> observation vector (not normalised)."""
    u = (np.asarray(q, float) - fxycxy[2:4]) / fxycxy[0:2]
    n2 = (u * u).sum(-1, keepdims=True)
    return np.concatenate((u, 1. - 0.25 * n2), -1)


def _unproject(q, lensmodel, intrinsics_data):
    if lensmodel == "LENSMODEL_STEREOGRAPHIC":
        return _unproject_stereographic(q, intrinsics_data)
    if lensmodel == "LENSMODEL_PINHOLE":
        u = (np.asarray(q, float) - intrinsics_data[2:4]) / intrinsics_data[0:2]
        return np.concatenate((u, np.ones(u.shape[:-1] + (1,))), -1)
    from . import api   # any other model: the library's unproject (GPU)
    return api.unproject(q, lensmodel, intrinsics_data)


# --------------------------------------------------------------------------- PnP for a planar target
class _PnPNegZ(Exception):
    pass


class _PnPTooFew(Exception):
    pass


def _pnp_planar(obj, q, fxy, cxy):
    """Pose Rt_cam_obj of a planar target (obj: (N,3) with z=0, q: (N,2) pinhole pixels)."""
    x = (q - cxy) / fxy                      # normalised image coordinates
    X = obj[:, :2]
    # normalise for conditioning (Hartley)
    mX, sX = X.mean(0), X.std() + 1e-12
    mx, sx = x.mean(0), x.std() + 1e-12
    Xn, xn = (X - mX) / sX, (x - mx) / sx
    N = X.shape[0]
    A = np.zeros((2 * N, 9))
    A[0::2, 0:2] = Xn; A[0::2, 2] = 1.; A[0::2, 6:8] = -xn[:, :1] * Xn; A[0::2, 8] = -xn[:, 0]
    A[1::2, 3:5] = Xn; A[1::2, 5] = 1.; A[1::2, 6:8] = -xn[:, 1:] * Xn; A[1::2, 8] = -xn[:, 1]
    Hn = np.linalg.svd(A)[2][-1].reshape(3, 3)
    TX = np.array(((1 / sX, 0, -mX[0] / sX), (0, 1 / sX, -mX[1] / sX), (0, 0, 1.)))
    Tx = np.array(((sx, 0, mx[0]), (0, sx, mx[1]), (0, 0, 1.)))
    Hm = Tx @ Hn @ TX
    # H ~ [r1 r2 t]
    s = 2. / (np.linalg.norm(Hm[:, 0]) + np.linalg.norm(Hm[:, 1]))
    Hm = Hm * s
    if Hm[2, 2] < 0:
        Hm = -Hm
    r1, r2, t = Hm[:, 0], Hm[:, 1], Hm[:, 2]
    U, _, Vt = np.linalg.svd(np.stack((r1, r2, np.cross(r1, r2)), 1))
    R = U @ Vt
    if np.linalg.det(R) < 0:
        R = U @ np.diag((1., 1., -1.)) @ Vt
    rt = np.concatenate((r_from_R(R), t))
    return _pnp_refine(obj, x, rt)


def _pnp_refine(obj, x, rt, iterations=20):
    """Gauss-Newton on the normalised-pinhole reprojection error, numerical Jacobian (6 unknowns)."""
    def res(rt):
        p = obj @ R_from_r(rt[:3]).T + rt[3:]
        return (p[:, :2] / p[:, 2:3] - x).ravel()
    lam = 1e-6
    r0 = res(rt)
    for _ in range(iterations):
        J = np.zeros((r0.size, 6))
        for k in range(6):
            d = np.zeros(6); d[k] = 1e-6
            J[:, k] = (res(rt + d) - r0) / 1e-6
        H = J.T @ J
        step = np.linalg.solve(H + lam * np.diag(np.diag(H) + 1e-12), -J.T @ r0)
        r1 = res(rt + step)
        if r1 @ r1 < r0 @ r0:
            rt, r0, lam = rt + step, r1, max(lam / 10., 1e-12)
            if np.linalg.norm(step) < 1e-12:
                break
        else:
            lam *= 10.
            if lam > 1e6:
                break
    return rt


def _estimate_camera_pose_from_fixed_point_observations(lensmodel, intrinsics_data, observation_qxqyw, points_ref, what):
    """mrcal/calibration.py:508-620: unproject through the given model, re-project through a pinhole of
    (scaled) focal length, solve the planar PnP; retry with a longer / shorter focal length if the target
    lands behind the camera / too few points survive."""
    intrinsics_data = np.asarray(intrinsics_data, float)

    def attempt(scale):
        fxy, cxy = intrinsics_data[0:2], intrinsics_data[2:4]
        v = _unproject((observation_qxqyw[..., :2] - cxy) / scale + cxy, lensmodel, intrinsics_data)
        with np.errstate(divide="ignore", invalid="ignore"):
            q_pinhole = v[..., :2] / v[..., 2:3] * fxy + cxy
        q_pinhole = q_pinhole * scale + cxy * (1. - scale)
        ok = (observation_qxqyw[..., 2] > 0.0) & np.isfinite(v).all(-1) & np.isfinite(q_pinhole).all(-1) & (v[..., 2] > 0)
        if np.count_nonzero(ok) < 6:
            raise _PnPTooFew(f"Insufficient observations; need at least 6; got {np.count_nonzero(ok)} instead. "
                             f"Cannot estimate initial extrinsics for {what}")
        rt = _pnp_planar(points_ref[ok], q_pinhole[ok], fxy * scale, cxy)
        if rt[5] <= 0:
            # the mirror solution: flip through the origin and refine again
            rt2 = rt.copy()
            rt2[3:] = -rt2[3:]
            rt = _pnp_refine(points_ref[ok], (q_pinhole[ok] - cxy) / (fxy * scale), rt2)
            if rt[5] <= 0:
                raise _PnPNegZ(f"The chessboard ends up behind the camera. Cannot estimate initial extrinsics for {what}")
        return Rt_from_rt(rt)

    try:
        return attempt(1.)
    except _PnPNegZ:
        return attempt(1.5)
    except _PnPTooFew:
        return attempt(0.7)


def estimate_monocular_calobject_poses_Rt_tocam(indices_frame_camera, observations, object_spacing,
                                                models_or_intrinsics, *, paths=None):
    """Camera-referenced pose of the board in every observation: (Nobservations,4,3) Rt transforms TO the camera
    FROM the board (mrcal/calibration.py:622-781). models_or_intrinsics: per camera, a (lensmodel,
    intrinsics_data) tuple or an object with .intrinsics()."""
    li = [m.intrinsics() if hasattr(m, "intrinsics") else m for m in models_or_intrinsics]
    H, W = observations.shape[-3:-1]
    points_ref = ref_calibration_object(W, H, object_spacing).reshape(-1, 3)
    obs = np.asarray(observations, float).reshape(observations.shape[0], -1, 3)
    out = np.zeros((obs.shape[0], 4, 3))
    for i in range(obs.shape[0]):
        icam = int(indices_frame_camera[i, 1])
        note = "" if paths is None else f'; "{paths[i]}"'
        out[i] = _estimate_camera_pose_from_fixed_point_observations(
            li[icam][0], li[icam][1], obs[i], points_ref, f"observation {i} (camera {icam}{note})")
    return out


# --------------------------------------------------------------------------- camera poses
def traverse_sensor_links(connectivity_matrix, callback_sensor_link):
    """Visit the sensors in order of distance from sensor 0 over the graph whose edge cost is
    65536 - (shared frames) (traverse-sensor-links.c:17-24), calling callback_sensor_link(idx, idx_parent) when
    the best path to a sensor is known. Sensors not connected to sensor 0 are never visited."""
    C = np.asarray(connectivity_matrix)
    N = C.shape[0]
    cost = [None] * N
    parent = [-1] * N
    done = [False] * N
    heap = []

    def visit(i):
        done[i] = True
        for j in range(N):
            if j == i or C[i, j] == 0 or done[j]:
                continue
            c = cost[i] + (65536 - int(C[i, j]))
            if cost[j] is None or c < cost[j]:
                cost[j] = c
                parent[j] = i
                heapq.heappush(heap, (c, j))

    cost[0] = 0
    visit(0)
    while heap:
        c, j = heapq.heappop(heap)
        if done[j] or c != cost[j]:
            continue
        callback_sensor_link(j, parent[j])
        visit(j)


def _estimate_camera_poses(calobject_poses_local_Rt_cf, indices_frame_camera, object_width_n, object_height_n, object_spacing):
    """Rt_0c of every camera but the first (mrcal/calibration.py:925-1101): pairwise alignment of the board as
    seen by the two cameras of a link, over the frames both see; links chosen by traverse_sensor_links()."""
    ifc = np.asarray(indices_frame_camera)
    Ncameras = int(ifc[:, 1].max()) + 1
    Rt_0c = [None] * (Ncameras - 1)
    ref_object = ref_calibration_object(object_width_n, object_height_n, object_spacing).reshape(-1, 3)

    def compute_pairwise_Rt(icam_to, icam_from):
        if icam_to > icam_from:
            return invert_Rt(compute_pairwise_Rt(icam_from, icam_to))
        if icam_to == icam_from:
            raise RuntimeError(f"Got icam_to == icam_from ( = {icam_to} ). This was probably a mistake")
        A, B = [], []
        iframe_last, Rt0 = -1, None
        for i in range(ifc.shape[0]):
            iframe, icam = ifc[i]
            if iframe != iframe_last:
                Rt0, iframe_last = None, iframe
            if icam == icam_to:
                Rt0 = calobject_poses_local_Rt_cf[i]
            elif icam == icam_from and Rt0 is not None:
                A.append(transform_point_Rt(Rt0, ref_object))
                B.append(transform_point_Rt(calobject_poses_local_Rt_cf[i], ref_object))
        return align_procrustes_points_Rt01(np.concatenate(A), np.concatenate(B))

    shared = np.zeros((Ncameras, Ncameras), np.int64)
    for f in np.unique(ifc[:, 0]):
        cams = ifc[ifc[:, 0] == f, 1]
        for a in range(len(cams)):
            for b in range(a + 1, len(cams)):
                shared[cams[a], cams[b]] += 1
                shared[cams[b], cams[a]] += 1
    shared[shared < 2] = 0   # align_procrustes needs overlap

    def found_best_path_to_node(camera_idx, from_idx):
        Rt_fc = compute_pairwise_Rt(from_idx, camera_idx)
        Rt_0c[camera_idx - 1] = Rt_fc if from_idx == 0 else compose_Rt(Rt_0c[from_idx - 1], Rt_fc)

    traverse_sensor_links(shared, found_best_path_to_node)
    if any(x is None for x in Rt_0c):
        raise RuntimeError("ERROR: Don't have complete camera observations overlap!\n"
                           f"Shared observations matrix:\n{shared}\n")
    return np.array(Rt_0c).reshape(-1, 4, 3)


def estimate_joint_frame_poses(calobject_Rt_camera_frame, Rt_cam_ref, indices_frame_camera,
                               object_width_n, object_height_n, object_spacing):
    """rt_ref_frame (Nframes,6): per frame, the board pose in the reference frame; with several observing cameras,
    the pose that best fits the mean of the per-camera estimates of the corner positions
    (mrcal/calibration.py:1186-1396)."""
    ifc = np.asarray(indices_frame_camera)
    Rt_ref_cam = invert_Rt(np.asarray(Rt_cam_ref, float).reshape(-1, 4, 3)) if len(Rt_cam_ref) else np.zeros((0, 4, 3))
    obj = ref_calibration_object(object_width_n, object_height_n, object_spacing).reshape(-1, 3)

    def single(i):
        icam = int(ifc[i, 1])
        Rt = calobject_Rt_camera_frame[i]
        return Rt if icam == 0 else compose_Rt(Rt_ref_cam[icam - 1], Rt)

    out = []
    i0 = 0
    for i in range(1, ifc.shape[0] + 1):
        if i == ifc.shape[0] or ifc[i, 0] != ifc[i0, 0]:
            if i - i0 == 1:
                Rt = single(i0)
            else:
                mean = sum(transform_point_Rt(single(k), obj) for k in range(i0, i)) / (i - i0)
                Rt = align_procrustes_points_Rt01(mean, obj)
            out.append(rt_from_Rt(Rt))
            i0 = i
    return np.array(out).reshape(-1, 6)


def seed_stereographic(imagersizes, focal_estimate, indices_frame_camera, observations, object_spacing, *, paths=None):
    """A seed for a calibration solve: (intrinsics_data (Ncameras,4), rt_cam_ref (Ncameras-1,6),
    rt_ref_frame (Nframes,6)) for LENSMODEL_STEREOGRAPHIC with the given focal-length guess and the imager centre
    as the projection centre (mrcal/calibration.py:1398-1608)."""
    Ncameras = len(imagersizes)
    try:
        focal = list(focal_estimate)
    except TypeError:
        focal = [focal_estimate]
    if len(focal) == 1:
        focal = focal * Ncameras
    elif len(focal) != Ncameras:
        raise RuntimeError(f"Ncameras mismatch: len(imagersizes) = {Ncameras} but len(focal_estimate) = {len(focal)}")
    intrinsics = [("LENSMODEL_STEREOGRAPHIC",
                   np.array((focal[i], focal[i], (imagersizes[i][0] - 1.) / 2., (imagersizes[i][1] - 1.) / 2.)))
                  for i in range(Ncameras)]
    Rt_cf = estimate_monocular_calobject_poses_Rt_tocam(indices_frame_camera, observations, object_spacing,
                                                        intrinsics, paths=paths)
    H, W = observations.shape[-3:-1]
    Rt_0c = _estimate_camera_poses(Rt_cf, indices_frame_camera, W, H, object_spacing)
    Rt_cam_ref = invert_Rt(Rt_0c) if len(Rt_0c) else np.zeros((0, 4, 3))
    rt_ref_frame = estimate_joint_frame_poses(Rt_cf, Rt_cam_ref, indices_frame_camera, W, H, object_spacing)
    rt_cam_ref = rt_from_Rt(Rt_cam_ref).reshape(-1, 6) if len(Rt_cam_ref) else np.zeros((0, 6))
    return np.array([i[1] for i in intrinsics]), rt_cam_ref, rt_ref_frame
