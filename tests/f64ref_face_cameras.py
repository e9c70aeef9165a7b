"""Plain float64 restatement of g2pc_face_cameras (normals turned toward the camera that saw each Gaussian;
g2pc/orient.py face_cameras, gauss_to_mesh.py; rules in DESIGN.md §2), and hand cases with known outcomes."""
import numpy as np

INT32_MAX = 2 ** 31 - 1


def face_cameras(means, normals, ids, cam_of, cams):
    """Normals turned toward the camera that saw each Gaussian (g2pc_face_cameras; rules in DESIGN.md §2).  Returns (out:
    the normals with the flipped rows negated, counts [flipped, unseen, undecided, invalid]).  Row r: f = cam_of[ids[r]];
    invalid when ids[r] is outside [0, N) or f is outside [0, ncam) and not INT32_MAX, unseen when f == INT32_MAX;
    otherwise dot = (nx*dx + ny*dy) + nz*dz, d = c_f - mu, in float64: flipped when dot < 0, undecided when dot == 0 or
    NaN."""
    mu = np.asarray(means, np.float32).astype(np.float64).reshape(-1, 3)
    nrm = np.asarray(normals)
    n64 = nrm.astype(np.float64)
    ids = np.asarray(ids, np.int64)
    cam_of = np.asarray(cam_of, np.int64)
    c = np.asarray(cams, np.float32).astype(np.float64).reshape(-1, 3)
    okid = (ids >= 0) & (ids < cam_of.shape[0])
    f = np.full(ids.shape, -1, np.int64)
    f[okid] = cam_of[ids[okid]]
    unseen = okid & (f == INT32_MAX)
    invalid = ~okid | (~unseen & ((f < 0) | (f >= c.shape[0])))
    seen = ~(invalid | unseen)
    d = c[f[seen]] - mu[seen]
    with np.errstate(invalid="ignore", over="ignore"):
        dot = (n64[seen, 0] * d[:, 0] + n64[seen, 1] * d[:, 1]) + n64[seen, 2] * d[:, 2]
    flip = np.zeros(ids.shape, bool)
    flip[seen] = dot < 0
    undecided = np.zeros(ids.shape, bool)
    undecided[seen] = ~((dot < 0) | (dot > 0))
    out = nrm.copy()
    out[flip] = -out[flip]
    return out, np.array([flip.sum(), unseen.sum(), undecided.sum(), invalid.sum()], np.int64)


def face_camera_hand_cases(dtype):
    """(means, normals, ids, cam_of, cams, expected flip mask, expected counts) of rows with known outcomes: a dot of
    exactly 0, a camera at the Gaussian's centre, +-0 components, NaN / Inf / zero normals, unseen and invalid rows."""
    cams = np.float32([[0, 0, 10], [5, 0, 0], [1, 2, 3]])
    N = 12
    cam_of = np.full(N, INT32_MAX, np.int64)
    rows = []  # (mean, normal, id, class: 0 flipped, 1 unseen, 2 undecided, 3 invalid, 4 kept)

    def row(mean, nrm, cam, cls):  # a row with its own id, whose camera is cam (None: unseen)
        g = len(rows)
        if cam is not None:
            cam_of[g] = cam
        rows.append((mean, nrm, g, cls))

    row([0, 0, 0], [0, 0, 1], 0, 4)             # faces camera 0
    row([0, 0, 0], [0, 0, -1], 0, 0)            # away from camera 0
    row([0, 0, 0], [1, 0, 0], 0, 2)             # perpendicular: dot exactly 0
    row([1, 2, 3], [0, 0, -1], 2, 2)            # camera at the centre: d = 0
    row([0, 0, 0], [-0.0, 0.0, -1], 0, 0)       # +-0 components, flipped: the zeros change sign
    row([0, 0, 0], [-0.0, -0.0, 0.0], 1, 2)     # zero normal
    row([0, 0, 0], [np.nan, 0, 1], 0, 2)        # NaN
    row([0, 0, 0], [0, 0, -np.inf], 0, 0)       # -Inf toward away: -Inf * 10 < 0
    row([0, 0, 0], [np.inf, 0, 0], 0, 2)        # Inf * 0 = NaN
    row([0, 0, 0], [0, 0, 1], None, 1)          # unseen
    row([0, 0, 0], [0, 0, 1], 3, 3)             # camera index out of range
    row([0, 0, 0], [0, 0, 1], -1, 3)            # negative camera index
    rows.append(([0, 0, 0], [0, 0, 1], N, 3))   # id out of range
    rows.append(([0, 0, 0], [0, 0, 1], -1, 3))  # negative id
    means = np.float32([r[0] for r in rows])
    nrm = np.array([r[1] for r in rows], dtype)
    ids = np.int32([r[2] for r in rows])
    cls = np.array([r[3] for r in rows])
    counts = np.array([(cls == k).sum() for k in range(4)], np.int64)
    return means, nrm, ids, cam_of.astype(np.int32), cams, cls == 0, counts
