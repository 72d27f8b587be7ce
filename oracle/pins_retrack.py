"""Inputs of the motion-hypothesis pin (SURVEY.md 8f n6): the scene, levels and trackers of oracle/pins_pyramid.py, plus try
lists and lastCoarseRMSE values for five cases.

motion_tries() builds lastF_2_fh_tries the way FullSystem::trackNewCoarse does (FullSystem.cpp:437-534): five motion models and
26 small rotations around the constant-motion guess.  It is a test-input generator only and is NOT pinned: the reference loop,
the restatement and the device all receive the same list, so the loop is pinned whatever the list holds."""
import numpy as np

from oracle import pins_pyramid as P
from oracle.lm_driver import hat, se3_exp

# (x, y, z) signs of the 26 rotation tries, in the order of :454-529 (quaternion (1, x rotDelta, y rotDelta, z rotDelta))
ROT_SIGNS = ((1, 0, 0), (0, 1, 0), (0, 0, 1), (-1, 0, 0), (0, -1, 0), (0, 0, -1),
             (1, 1, 0), (0, 1, 1), (1, 0, 1), (-1, 1, 0), (0, -1, 1), (-1, 0, 1),
             (1, -1, 0), (0, 1, -1), (1, 0, -1), (-1, -1, 0), (0, -1, -1), (-1, 0, -1),
             (-1, -1, -1), (-1, -1, 1), (-1, 1, -1), (-1, 1, 1), (1, -1, -1), (1, -1, 1), (1, 1, -1), (1, 1, 1))


def se3_log(T):
    """Inverse of lm_driver.se3_exp (Sophus convention (upsilon, omega)); rotation angles below pi."""
    R = np.asarray(T, np.float64)[:3, :3]
    c = np.clip((np.trace(R) - 1) / 2, -1.0, 1.0)
    th = np.arccos(c)
    w = np.array([R[2, 1] - R[1, 2], R[0, 2] - R[2, 0], R[1, 0] - R[0, 1]])
    om = w * (0.5 if th < 1e-8 else th / (2 * np.sin(th)))
    Om = hat(om)
    if th < 1e-8:
        Vi = np.eye(3) - 0.5 * Om + Om @ Om / 12
    else:
        Vi = np.eye(3) - 0.5 * Om + (1 - th * np.sin(th) / (2 * (1 - np.cos(th)))) / th ** 2 * Om @ Om
    return np.concatenate([Vi @ np.asarray(T, np.float64)[:3, 3], om])


def quat_pose(w, x, y, z):
    """SE3(Sophus::Quaterniond(w, x, y, z), 0): the quaternion is normalised."""
    q = np.array([w, x, y, z], np.float64)
    w, x, y, z = q / np.linalg.norm(q)
    T = np.eye(4)
    T[:3, :3] = [[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                 [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                 [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]]
    return T


def motion_tries(fh_2_slast, lastF_2_slast, pose_valid=True):
    """lastF_2_fh_tries of FullSystem.cpp:437-534 as (n, 4, 4): constant, double, half and zero motion, zero motion from the
    keyframe, then the 26 rotations by rotDelta = 0.02f around the constant-motion guess; [identity] when a pose is invalid."""
    if not pose_valid:
        return np.eye(4)[None].copy()
    inv = np.linalg.inv
    f, l = np.asarray(fh_2_slast, np.float64), np.asarray(lastF_2_slast, np.float64)
    const = inv(f) @ l
    out = [const, inv(f) @ inv(f) @ l, inv(se3_exp(se3_log(f) * 0.5)) @ l, l.copy(), np.eye(4)]
    d = float(np.float32(0.02))
    for x, y, z in ROT_SIGNS:
        out.append(const @ quat_pose(1.0, x * d, y * d, z * d))
    return np.stack(out)


def _motion(tx, ty, tz, rx=0.0, ry=0.0, rz=0.0):
    return se3_exp([tx, ty, tz, rx, ry, rz])


def case_inputs(name):
    """(tries (n, 4, 4), last_coarse_rmse (5,), call arguments of track_pyramid for every try)."""
    c = CASES[name]
    _, _, _, T_true = P.scene()
    return c["tries"](T_true), np.full(5, c["last_rmse"]), c["args"]


DSO = dict(coarse_cutoff=20.0, new_exposure=1.05, mode_a=1e12, mode_b=1e8)   # settings.cpp:109-110 modes
# Start poses around the true pose T (left-multiplied) and their outcome on this scene (CPU oracle, 320x240, 4 levels, DSO)
LOCAL_MIN = (-0.057, -0.181, -0.246, 0.064, -0.161, 0.138)   # ok at a local minimum: lastResiduals about 9.8 9.7 9.4 9.2
FAR = _motion(0.25, -0.1, 0.2, 0.0, 0.25, 0.0)              # a last motion far larger than the true one: the constant, double
                                                             # and rotated guesses end level 3 near 15-16.5, the half-motion
                                                             # guess converges to the truth


def _around(T, *xis):
    return np.stack([se3_exp(xi) @ T for xi in xis])


# name -> tries(T_true), lastCoarseRMSE (all five levels), track arguments; tests/test_track_new_coarse_cpu.py asserts what each
# case is named for
CASES = {
    # lastCoarseRMSE.setConstant(100) (:154): the constant-motion guess is the truth, wins and the loop stops after one try
    "first": dict(tries=lambda T: motion_tries(_motion(0.01, 0, 0), _motion(0.01, 0, 0) @ T), last_rmse=100.0, args=DSO),
    # try 0 wins at a local minimum (no break: 9.8 >= 4 * 1.5), the constant and double motion guesses abort on level 3,
    # the half-motion guess wins with the true pose and stops the loop before the last two tries
    "retrack": dict(tries=lambda T: np.concatenate([_around(T, LOCAL_MIN), motion_tries(FAR, T)[:5]]), last_rmse=4.0, args=DSO),
    # lastCoarseRMSE = 0: every try runs.  Try 0 wins at the local minimum, try 1 (constant motion) aborts on level 3, try 2
    # (half motion) wins with the true pose; tries 3 (the truth-start guess of "first") and 4 (zero motion) are ok but do not win
    # (lastResiduals[0] 3.01603 >= 3.01593), and take over achievedRes[1] (2.86398 < 2.86508): the takeover of :595-602 by tries
    # that are not winners.  Level 4 is never reached and stays NaN.
    "exhaust": dict(tries=lambda T: np.concatenate([_around(T, LOCAL_MIN), motion_tries(FAR, T)[[0, 2]],
                                                    motion_tries(_motion(0.01, 0, 0), _motion(0.01, 0, 0) @ T)[:1],
                                                    motion_tries(FAR, T)[[3]]]), last_rmse=0.0, args=DSO),
    # exposure ratio e^2 with the DSO priors: every try is rejected by |a| > 1.2 (:923-924)
    "none_good": dict(tries=lambda T: motion_tries(_motion(0.01, 0, 0), _motion(0.01, 0, 0) @ T)[:3], last_rmse=100.0,
                      args=dict(DSO, new_exposure=float(np.exp(2.0)))),
    # a pose of the history is invalid (:531-534): the list is [identity]
    "single": dict(tries=lambda T: motion_tries(None, None, pose_valid=False), last_rmse=100.0, args=DSO),
}
