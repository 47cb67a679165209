"""CPU: the answers the pose-utility GPU tests compare against (tests/poseutils_np.py and the stored
tests/golden/poseutils.npz), and the refusals that come before any device work."""
import numpy as np
import pytest

import mrcal_b200
import poseutils_np as U


def test_golden_matches_the_compiled_reference(ref):
    z = np.load(U.GOLDEN)
    for key, fname, args, kw, _ in U.cases():
        for k, a in enumerate(args):
            assert np.array_equal(z[f"{key}/in{k}"], a), key
        for k, a in enumerate(U.reference(fname, args, kw)):
            assert np.array_equal(z[f"{key}/out{k}"], a, equal_nan=True), f"{key} output {k}"


def test_quaternion_restatement_matches_scipy():
    from scipy.spatial.transform import Rotation
    rng = np.random.default_rng(1)
    R = Rotation.random(200, random_state=2).as_matrix()
    # every branch of the formula: near-identity, and half-turns about each axis
    R = np.concatenate((R, [np.eye(3), np.diag([1., -1, -1]), np.diag([-1., 1, -1]), np.diag([-1., -1, 1])]))
    q = U.quat_from_R(R)
    q_scipy = Rotation.from_matrix(R).as_quat()          # (x,y,z,w)
    q_scipy = np.concatenate((q_scipy[:, 3:], q_scipy[:, :3]), -1)
    # the same rotation: equal up to the sign of the whole quaternion
    sign = np.sign(np.sum(q * q_scipy, axis=-1))[:, None]
    assert np.abs(q - sign * q_scipy).max() < 1e-14
    assert np.abs(U.R_from_quat(q) - R).max() < 1e-14
    qr = rng.normal(size=(50, 4))
    qr /= np.linalg.norm(qr, axis=-1, keepdims=True)
    assert np.abs(U.R_from_quat(qr) - Rotation.from_quat(np.concatenate((qr[:, 1:], qr[:, :1]), -1))
                  .as_matrix()).max() < 1e-14


def test_skew_symmetric_restatement_is_the_cross_product():
    a, b = np.random.default_rng(3).normal(size=(2, 10, 3))
    assert np.abs(np.einsum("nij,nj->ni", U.skew_symmetric(a), b) - np.cross(a, b)).max() < 1e-14


def test_refusals_before_device_work():
    with pytest.raises(ValueError, match=r"shape \(\.\.\.,6\)"):
        mrcal_b200.transform_point_rt(np.zeros(5), np.zeros(3))
    with pytest.raises(ValueError, match=r"shape \(\.\.\.,3,3\)"):
        mrcal_b200.r_from_R(np.zeros((4, 3)))
    with pytest.raises(ValueError, match="do not broadcast"):
        mrcal_b200.transform_point_rt(np.zeros((2, 6)), np.zeros((3, 3)))
    with pytest.raises(ValueError, match=r"out must have shape \(4, 3\)"):
        mrcal_b200.rotate_point_r(np.zeros(3), np.zeros((4, 3)), out=np.zeros((3, 3)))
    with pytest.raises(ValueError, match="out must be a tuple of 3"):
        mrcal_b200.rotate_point_r(np.zeros(3), np.zeros(3), get_gradients=True, out=np.zeros(3))
    with pytest.raises(Exception, match="exactly 2 inputs"):
        mrcal_b200.compose_rt(np.zeros(6), np.zeros(6), np.zeros(6), get_gradients=True)
    with pytest.raises(Exception, match="exactly 2 inputs"):
        mrcal_b200.compose_r(np.zeros(3), np.zeros(3), np.zeros(3), inverted0=True)
    torch = pytest.importorskip("torch")
    with pytest.raises(RuntimeError, match="may not be mixed"):
        mrcal_b200.compose_rt(np.zeros(6), torch.zeros(6, dtype=torch.float64))
    with pytest.raises(ValueError, match="CUDA float64"):
        mrcal_b200.R_from_r(torch.zeros(3, dtype=torch.float64))


def test_identities_are_host_only():
    assert np.array_equal(mrcal_b200.identity_Rt(), np.vstack((np.eye(3), np.zeros((1, 3)))))
    assert np.array_equal(mrcal_b200.identity_rt(), np.zeros(6))
    out = np.ones((3, 3))
    assert mrcal_b200.identity_R(out=out) is out and np.array_equal(out, np.eye(3))
