"""Gaussian file I/O — thin host-side counterpart of the reference's gauss_dataloader.py (same function names).

Reference: gauss_dataloader.py (load_ply_data :16-82, load_splat_data :84-115, save_xyz_to_ply :118-202,
load_gaussians :204-211).  Outside the timed hot path (SURVEY.md §2 row 12, §8f N3): a small numpy PLY reader replaces the
`plyfile` dependency, and the PLY vertex records are assembled on the GPU (byte views of the f32 / u8 tensors) so the
point cloud crosses PCIe once, already in file layout.
"""
import os

import numpy as np
import torch

SH_C0 = 0.28209479177387814
_PLY_DTYPES = {"char": "i1", "uchar": "u1", "short": "i2", "ushort": "u2", "int": "i4", "uint": "u4", "float": "f4",
               "double": "f8", "int8": "i1", "uint8": "u1", "int16": "i2", "uint16": "u2", "int32": "i4", "uint32": "u4",
               "float32": "f4", "float64": "f8"}


def computeColorFromLowDegSH(sh):
    """DC colour: clip(C0 * sh[:, :, 0] + 0.5, 0, 1), f64 (gauss_dataloader.py:8-14)."""
    return ((SH_C0 * sh[:, :, 0].to(torch.double)) + 0.5).clip(0, 1).type(torch.double)


def read_ply_vertices(path):
    """Vertex element of a PLY file (ascii or binary little/big endian) as a numpy structured array."""
    with open(path, "rb") as f:
        if f.readline().strip() != b"ply":
            raise AttributeError(f"{path} is not a PLY file")
        fmt, props, count, in_vertex = None, [], 0, False
        while True:
            line = f.readline()
            if not line:
                raise AttributeError("unterminated PLY header")
            tok = line.decode("ascii", "replace").strip().split()
            if not tok:
                continue
            if tok[0] == "format":
                fmt = tok[1]
            elif tok[0] == "element":
                in_vertex = tok[1] == "vertex"
                if in_vertex:
                    count = int(tok[2])
            elif tok[0] == "property" and in_vertex:
                if tok[1] == "list":
                    raise AttributeError("list properties on the vertex element are not supported")
                props.append((tok[2], _PLY_DTYPES[tok[1]]))
            elif tok[0] == "end_header":
                break
        if fmt == "ascii":
            data = np.loadtxt(f, max_rows=count, ndmin=2)
            out = np.zeros(count, dtype=[(n, t) for n, t in props])
            for i, (n, _) in enumerate(props):
                out[n] = data[:, i]
            return out
        endian = "<" if fmt == "binary_little_endian" else ">"
        dt = np.dtype([(n, endian + t) for n, t in props])
        return np.frombuffer(f.read(count * dt.itemsize), dtype=dt, count=count)


def load_ply_data(path, max_sh_degree=3, device="cuda:0"):
    """Gaussians from a 3DGS .ply: xyz f32, log-scales f64, normalised quaternions f64, sigmoid opacities f32, SH
    (N,3,K) f64 channel-major and DC colours — or plain RGB columns (gauss_dataloader.py:16-82)."""
    v = read_ply_vertices(path)
    names = v.dtype.names
    xyz = np.stack((v["x"], v["y"], v["z"]), axis=1)
    opac = np.asarray(v["opacity"], dtype=np.float64)
    if "f_dc_0" in names:
        dc = np.stack([v["f_dc_0"], v["f_dc_1"], v["f_dc_2"]], axis=1).astype(np.float64)[:, :, None]
        rest_names = sorted((n for n in names if n.startswith("f_rest_")), key=lambda s: int(s.split("_")[-1]))
        assert len(rest_names) == 3 * (max_sh_degree + 1) ** 2 - 3
        rest = np.stack([v[n] for n in rest_names], axis=1).astype(np.float64) if rest_names else np.zeros((xyz.shape[0], 0))
        rest = rest.reshape(xyz.shape[0], 3, (max_sh_degree + 1) ** 2 - 1)
        features_all = torch.cat((torch.tensor(dc, device=device), torch.tensor(rest, device=device)), 2)
        colours = computeColorFromLowDegSH(features_all)
    elif "red" in names:
        colours = torch.tensor(np.stack([v["red"], v["green"], v["blue"]], axis=1).astype(np.float64), device=device)
        if torch.count_nonzero(colours > 1.0) > 0:
            colours = (colours / 255).clip(0, 1)
        features_all = None
    else:
        raise AttributeError("Input ply file does not have valid colours (must have either spherical harmoics or RGB colour fields)")
    scale_names = sorted((n for n in names if n.startswith("scale_")), key=lambda s: int(s.split("_")[-1]))
    rot_names = sorted((n for n in names if n.startswith("rot")), key=lambda s: int(s.split("_")[-1]))
    scales = np.stack([v[n] for n in scale_names], axis=1).astype(np.float64)
    rots = np.stack([v[n] for n in rot_names], axis=1).astype(np.float64)
    rots = rots / np.expand_dims(np.linalg.norm(rots, axis=1), 1)
    opacities = (1 / (1 + torch.exp(torch.tensor(-opac, device=device)))).type(torch.float)
    return (torch.tensor(np.ascontiguousarray(xyz), device=device), torch.tensor(scales, device=device),
            torch.tensor(rots, device=device), colours, opacities, features_all)


def load_splat_data(path, device="cuda:0"):
    """32-byte .splat records: xyz f32x3, scales f32x3, rgba u8x4, rot u8x4 (gauss_dataloader.py:84-115)."""
    dt = np.dtype([("xyz", np.float32, 3), ("scales", np.float32, 3), ("colour", np.uint8, 4), ("rots", np.uint8, 4)])
    rec = np.fromfile(path, dtype=dt)
    return (torch.tensor(rec["xyz"], device=device), torch.tensor(np.log(rec["scales"]), device=device),
            torch.tensor((rec["rots"].astype(np.float32) - 128) / 128, device=device),
            torch.tensor(rec["colour"][:, :3] / 255, device=device), torch.tensor(rec["colour"][:, 3] / 255, device=device),
            None)


def load_gaussians(input_path, max_sh_degree=3):
    ext = os.path.splitext(input_path)[1]
    if ext == ".splat":
        return load_splat_data(input_path)
    if ext == ".ply":
        return load_ply_data(input_path, max_sh_degree=max_sh_degree)
    raise AttributeError(f"Unsupported input type {ext}")


def save_xyz_to_ply(xyz_points, filename, rgb_colors=None, normals_points=None, chunk_size=10**6, quiet=False):
    """Binary little-endian PLY with the reference's header and record layout (gauss_dataloader.py:118-202):
    x y z [nx ny nz] f4, red green blue u1.  Records are interleaved on the device; one D2H copy per chunk."""
    assert xyz_points.shape[1] == 3, "Input points should be in the format (N, 3)"
    n = xyz_points.shape[0]
    if rgb_colors is None:
        rgb_colors = torch.full((n, 3), 255, dtype=torch.uint8, device=xyz_points.device)
    props = "property float x\nproperty float y\nproperty float z\n"
    if normals_points is not None:
        props += "property float nx\nproperty float ny\nproperty float nz\n"
    header = ("ply\nformat binary_little_endian 1.0\n" + f"element vertex {n}\n" + props +
              "property uchar red\nproperty uchar green\nproperty uchar blue\nend_header\n")
    with open(filename, "wb") as f:
        f.write(header.encode("utf-8"))
        for s in range(0, n, chunk_size):
            e = min(s + chunk_size, n)
            parts = [xyz_points[s:e].to(torch.float32).contiguous().view(torch.uint8).view(e - s, 12)]
            if normals_points is not None:
                parts.append(normals_points[s:e].to(torch.float32).contiguous().view(torch.uint8).view(e - s, 12))
            parts.append(rgb_colors[s:e].to(torch.uint8))
            f.write(torch.cat(parts, dim=1).contiguous().cpu().numpy().tobytes())
