"""Helpers shared by the GPU tests of the Node constructor (ORB / FAST detector, use_feature_min_depth, point clouds, colour
input): parameters and re-initialisation, rendered frames, and node dumps compared bit for bit."""
import ctypes as C

import numpy as np

MAXK = 600


def params(detector=0, max_keypoints=MAXK, **kw):
    from rgbdslam_v2_b200._capi import default_params
    p = default_params()
    p.depth_cov_z0 = 2.0
    p.max_keypoints = max_keypoints
    p.feature_detector_type = detector
    for k, v in kw.items():
        setattr(p, k, v)
    return p


def reinit(fe, detector=0, **kw):
    p = params(detector, **kw)
    fe.params = p
    fe._check(fe.lib.rgbdslam_b200_init(0, C.byref(p)))


def make_detector(fe, detector, **kw):
    """detector_create takes the type of the current parameters; the handle keeps it."""
    reinit(fe, detector, **kw)
    return fe.detector_create()


def name(detector):
    return "FAST" if detector == 1 else "ORB"


def K4():
    from rgbdslam_v2_b200 import synth
    return (synth.FX, synth.FY, synth.CX, synth.CY)


def render(ks, n_poses=240):
    """(gray, depth) of poses ks of an n_poses-pose synthetic trajectory, frame k rendered with seed k"""
    from rgbdslam_v2_b200 import synth
    poses = synth.trajectory(n_poses)
    return [synth.render_frame(poses[k], seed=k) for k in ks]


def stack(frames):
    return np.stack([f[0] for f in frames]), np.stack([f[1] for f in frames])


def seq(n):
    """the first n frames of the 240-pose trajectory: gray, depth and the mask the reference derives from depth"""
    from oracle import orb_oracle
    gray, depth = stack(render(range(n)))
    return gray, depth, np.stack([orb_oracle.depth_to_mask(d) for d in depth])


def textured(h, w, n, seed=0, sigma=2.0):
    """n frames of dense texture: band-limited noise (uniform noise blurred with sigma) wrapped four times over 0..255"""
    import cv2
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        t = cv2.GaussianBlur(rng.random((h, w)).astype(np.float32), (0, 0), sigma)
        out.append((t * 1024 % 256).astype(np.uint8))
    return np.stack(out)


class UnboundOrb:
    """cv2 with the detector's cv::ORB(10000, ...) replaced by cv::ORB(10^6, ...), whose per-level quotas never bind here:
    the reference's glue in the oracle without the quotas (monkeypatched over orb_oracle.cv2)"""

    def __getattr__(self, name):
        import cv2
        return getattr(cv2, name)

    @staticmethod
    def ORB_create(*a, **kw):
        import cv2
        if a and a[0] == 10000:
            a = (10 ** 6,) + a[1:]
        return cv2.ORB_create(*a, **kw)


def node_dump(fe, handles):
    return [(fe.node_keypoints(h), *fe.node_download(h)) for h in handles]


def same_nodes(a, b):
    for (ka, da, xa), (kb, db, xb) in zip(a, b):
        if not (np.array_equal(ka, kb) and np.array_equal(da, db) and np.array_equal(xa.view(np.uint32), xb.view(np.uint32))):
            return False
    return len(a) == len(b)


def destroy(fe, handles):
    for h in handles:
        fe.node_destroy(h)
