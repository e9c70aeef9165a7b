"""Camera pose / intrinsics loaders — thin host-side counterpart of the reference's transform_dataloader.py.

Reference: transform_dataloader.py (COLMAP bin :115-167, COLMAP txt :169-205, transforms.json :207-277,
dispatch :280-299).  Host parsing only, outside the hot path (SURVEY.md §2 row 13).  Returns
({image name: 4x4 c2w nested list (OpenGL)}, {image name: [w, h, fx, fy]}).
"""
import json
import os
import struct

import numpy as np

_FLIP = np.diag([1.0, -1.0, -1.0, 1.0])


def qvec2rotmat(q):
    w, x, y, z = q
    return np.array([[1 - 2 * y * y - 2 * z * z, 2 * x * y - 2 * w * z, 2 * z * x + 2 * w * y],
                     [2 * x * y + 2 * w * z, 1 - 2 * x * x - 2 * z * z, 2 * y * z - 2 * w * x],
                     [2 * z * x - 2 * w * y, 2 * y * z + 2 * w * x, 1 - 2 * x * x - 2 * y * y]])


def convert_sfm_pose_to_nerf(transform):
    """COLMAP pose -> OpenGL c2w: inverse, then flip y and z (transform_dataloader.py:8-22)."""
    return np.linalg.inv(transform) @ _FLIP


def get_colmap_img_transform(elems):
    """(id, qw qx qy qz, tx ty tz, ...) -> c2w nested list.  The reference builds the matrix from the NEGATED quaternion
    and the translation before inverting (transform_dataloader.py:97-113)."""
    q = -np.array([float(v) for v in elems[1:5]])
    t = np.array([float(v) for v in elems[5:8]]).reshape(3, 1)
    m = np.concatenate([np.concatenate([qvec2rotmat(q), t], 1), np.array([[0.0, 0.0, 0.0, 1.0]])], 0)
    return convert_sfm_pose_to_nerf(m).tolist()


def _stem(name):
    return os.path.basename(str(name)).split(".")[0]


def load_colmap_bin_data(input_path, skip_rate=0):
    cams = {}
    with open(os.path.join(input_path, "cameras.bin"), "rb") as f:
        for _ in range(struct.unpack("<Q", f.read(8))[0]):
            e = struct.unpack("<iiQQdddd", f.read(56))
            if e[1] != 1:
                print("WARNING: Colmap cameras are a not Pinhole camera type. Rendered Colour quality might be impacted!")
            cams[e[0]] = e[2:]
    transforms, intr = {}, {}
    with open(os.path.join(input_path, "images.bin"), "rb") as f:
        for i in range(struct.unpack("<Q", f.read(8))[0]):
            e = struct.unpack("<idddddddi", f.read(64))
            name = b""
            while True:
                c = f.read(1)
                if c == b"":
                    raise EOFError("images.bin is truncated (image name not NUL-terminated)")
                if c == b"\x00":
                    break
                name += c
            npts = struct.unpack("<Q", f.read(8))[0]
            f.seek(24 * npts, 1)
            if i % (skip_rate + 1) == 0:
                key = _stem(name.decode("utf-8"))
                transforms[key] = get_colmap_img_transform(e)
                intr[key] = cams[e[8]]
    return transforms, intr


def load_colmap_txt_data(input_path, skip_rate=0):
    cams = {}
    with open(os.path.join(input_path, "cameras.txt")) as f:
        for line in f:
            line = line.strip()
            if not line or line[0] == "#":
                continue
            e = line.split(" ")
            if e[1].lower().strip() != "pinhole":
                print("WARNING: Colmap cameras are not a Pinhole camera type. Rendered Colour quality might be impacted!")
            cams[int(e[0])] = e[2:]
    transforms, intr = {}, {}
    i = 0
    with open(os.path.join(input_path, "images.txt")) as f:
        for line in f:
            line = line.strip()
            if line and line[0] == "#":
                continue
            i += 1
            if not line:
                continue
            if i % 2 == 1 and i % (skip_rate + 1) == 0:  # same selection rule as the reference (:190-192)
                e = line.split(" ")
                key = _stem(e[9])
                transforms[key] = get_colmap_img_transform(e)
                intr[key] = cams[int(e[8])]
    return transforms, intr


def get_transform_intrinsics(tr, fname):
    """[w, h, fx, fy] from a transforms.json block (transform_dataloader.py:207-243)."""
    out = [0, 0, 0, 0]
    if "w" in tr and "h" in tr:
        out[0], out[1] = tr["w"], tr["h"]
    else:
        if not os.path.exists(fname):
            raise Exception(f"Image with path {fname} does not exist")
        import cv2
        img = cv2.imread(fname)
        out[0], out[1] = img.shape[1], img.shape[0]
    if "fl_x" in tr:
        out[2] = tr["fl_x"]
    elif "camera_angle_x" in tr:
        out[2] = 0.5 * out[0] / np.tan(0.5 * tr["camera_angle_x"])
    else:
        raise Exception("A focal length (fl_x) or field of view (camera_angle_x) must be provided")
    if "fl_y" in tr:
        out[3] = tr["fl_y"]
    elif "camera_angle_y" in tr:
        out[3] = 0.5 * out[1] / np.tan(0.5 * tr["camera_angle_y"])
    else:
        out[3] = out[2]
    return out


def load_transform_json_data(input_path, skip_rate=0):
    with open(input_path) as f:
        tr = json.load(f)
    shared = None
    if "fl_x" in tr or "camera_angle_x" in tr:
        shared = get_transform_intrinsics(tr, tr["frames"][0]["file_path"])
    transforms, intr = {}, {}
    for i, frame in enumerate(tr["frames"]):
        key = _stem(frame["file_path"])
        intr[key] = shared if shared is not None else get_transform_intrinsics(frame, frame["file_path"])
        if i % (skip_rate + 1) == 0:
            transforms[key] = frame["transform_matrix"]
    return transforms, intr


def load_transform_data(input_path, skip_rate=0):
    if os.path.isdir(input_path):
        for base in (input_path, os.path.join(input_path, "sparse", "0")):
            if os.path.exists(os.path.join(base, "images.txt")):
                return load_colmap_txt_data(base, skip_rate=skip_rate)
            if os.path.exists(os.path.join(base, "images.bin")):
                return load_colmap_bin_data(base, skip_rate=skip_rate)
    elif os.path.splitext(input_path)[1] == ".json":
        return load_transform_json_data(input_path, skip_rate=skip_rate)
    raise AttributeError("Unsupported transform data type")
