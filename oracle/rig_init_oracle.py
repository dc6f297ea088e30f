"""ORACLE (test infrastructure, NOT product code) -- numpy restatement of ConvertRotationsFromImageToRig
(glomap/estimators/rotation_initializer.cc:7-125) under the rules of b200sfm_rig_rotations_from_images (include/b200sfm.h),
written as the reference's loops over frames and images, and of the numeric steps of SolveRotationAveraging's pre-pass for
rigs (controllers/rotation_averager.cc:81-182): the maximum spanning tree from oracle.mst_oracle, the rotation averages
from oracle.ra_oracle.  ``solve_rotation_averaging_rig`` runs the layout of glomap_b200.rotation_averager on those
numpy steps, so that the device chain can be compared with it step for step."""
from __future__ import annotations

import numpy as np

from oracle import mst_oracle, ra_oracle


def _qmul(a, b):
    """Eigen's quaternion product, xyzw."""
    ax, ay, az, aw = a
    bx, by, bz, bw = b
    return np.array([aw * bx + ax * bw + ay * bz - az * by, aw * by - ax * bz + ay * bw + az * bx,
                     aw * bz + ax * by - ay * bx + az * bw, aw * bw - ax * bx - ay * by - az * bz])


def _conj(q):
    return np.array([-q[0], -q[1], -q[2], q[3]])


def _unit(q):
    q = np.asarray(q, np.float64)
    return q / np.linalg.norm(q)


def average_quaternions(qs):
    """colmap::AverageQuaternions with unit weights (UPSTREAM-UNVERIFIED restatement): the eigenvector of sum q q^T with
    the largest eigenvalue over the normalised samples; a single sample as it is.  Canonical sign w >= 0."""
    qs = np.array([_unit(q) for q in qs])
    v = qs[0] if len(qs) == 1 else np.linalg.eigh(qs.T @ qs)[1][:, -1]
    v = v / np.linalg.norm(v)
    return -v if v[3] < 0 else v


def convert_rotations(image_frame, image_camera, cam_from_world, frame_ref_camera, camera_known, cam_from_rig,
                      rig_from_world, image_estimated=None):
    """Returns (cam_from_rig [K,4], cam_samples [K], rig_from_world [F,4], frame_samples [F]) like
    glomap_b200.rotation_initializer.convert_rotations_from_image_to_rig."""
    fr, cam = np.asarray(image_frame, np.int64), np.asarray(image_camera, np.int64)
    q = np.asarray(cam_from_world, np.float64).reshape(-1, 4)
    ref_cam, known = np.asarray(frame_ref_camera, np.int64), np.asarray(camera_known, bool)
    est = np.ones(len(fr), bool) if image_estimated is None else np.asarray(image_estimated, bool)
    cq = np.array(cam_from_rig, np.float64).reshape(-1, 4).copy()
    fq = np.array(rig_from_world, np.float64).reshape(-1, 4).copy()
    F, K = len(ref_cam), len(known)
    images_of = [[] for _ in range(F)]
    for i in range(len(fr)):                       # Frame::ImageIds(), registered images, ascending index
        if fr[i] >= 0:
            images_of[fr[i]].append(i)
    ref = np.full(F, -1, np.int64)
    samples = [[] for _ in range(K)]
    for f in range(F):                             # .cc:24-73
        for i in images_of[f]:
            if cam[i] == ref_cam[f]:
                ref[f] = i
                break
        r = ref[f]
        if r < 0:
            continue
        for i in images_of[f]:
            if cam[i] == ref_cam[f] or known[cam[i]] or not (est[i] and est[r]):
                continue
            samples[cam[i]].append(_qmul(_unit(q[i]), _conj(_unit(q[r]))))
    cn = np.array([len(s) for s in samples], np.int32)
    for c in range(K):                             # .cc:79-88
        if samples[c]:
            cq[c] = average_quaternions(samples[c])
    avail = known | (cn > 0)
    fn = np.zeros(F, np.int32)
    for f in range(F):                             # .cc:91-122
        s = []
        for i in images_of[f]:
            if not est[i]:
                continue
            if i == ref[f]:
                s.append(_unit(q[i]))
            elif avail[cam[i]]:
                s.append(_qmul(_conj(_unit(cq[cam[i]])), _unit(q[i])))
        fn[f] = len(s)
        if s:
            fq[f] = average_quaternions(s)
    return cq, cn, fq, fn


class OracleOps:
    """The numeric steps of glomap_b200.rotation_averager._solve_rig in numpy."""

    def __init__(self, options):
        self.opts = ra_oracle.RAOptions(
            max_num_l1_iterations=options.max_num_l1_iterations, l1_step_convergence_threshold=options.l1_step_convergence_threshold,
            max_num_irls_iterations=options.max_num_irls_iterations,
            irls_step_convergence_threshold=options.irls_step_convergence_threshold,
            irls_loss_parameter_sigma=options.irls_loss_parameter_sigma,
            weight_type="HALF_NORM" if options.weight_type == 1 else "GEMAN_MCCLURE", use_weight=options.use_weight)

    def mst(self, vg):
        R, parent, _ = mst_oracle.mst_init(vg.n_images, vg.ei, vg.ej, vg.R_rel, vg.weight, root=0)
        return R, parent >= 0

    def convert(self, *args, **kw):
        return convert_rotations(*args, **kw)

    def estimate(self, vg, R0):
        theta, info = ra_oracle.estimate_rotations(vg.n_images, vg.ei, vg.ej, vg.R_rel, ra_oracle.R_to_aa(R0), vg.weight,
                                                   self.opts)
        return not info.get("failed", False), ra_oracle.aa_to_R(theta), (info["l1_iterations"], info["irls_iterations"])

    def estimate_rig(self, g, R_frames0, R_cams0):
        nf = g["n_frames"]
        cfb = g["cam_frames_begin"]
        cam_frames = [g["cam_frames"][cfb[c]:cfb[c + 1]] for c in range(g["n_cams"])]
        theta0 = np.concatenate([ra_oracle.R_to_aa(R_frames0), ra_oracle.R_to_aa(R_cams0)])
        theta, info = ra_oracle.estimate_rotations_rig_unknown(nf, g["n_cams"], g["ei"], g["ej"], g["eci"], g["ecj"], g["R_rel"],
                                                               theta0, cam_frames, self.opts, edge_weight=g["weight"])
        R = ra_oracle.aa_to_R(theta)
        return True, R[:nf], R[nf:], (info["l1_iterations"], info["irls_iterations"])


def solve_rotation_averaging_rig(vg, image_frame, image_camera, camera_known, cam_from_rig, frame_ref_camera, options=None,
                                 R_init=None, info=None):
    """glomap_b200.rotation_averager.solve_rotation_averaging_rig on OracleOps."""
    import dataclasses

    from glomap_b200 import rotation_averager as RA
    o = options or RA.RotationAveragerOptions()
    est = RA.RotationEstimatorOptions(**{f.name: getattr(o, f.name) for f in dataclasses.fields(RA.RotationEstimatorOptions)})
    return RA._solve_rig(vg, image_frame, image_camera, camera_known, cam_from_rig, frame_ref_camera, o, R_init,
                         OracleOps(est), {} if info is None else info)
