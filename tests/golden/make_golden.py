"""Generate the golden vectors that pin the oracle and the kernels: outputs of the UNMODIFIED reference, on small
seeded scenes.  Inputs are regenerated from the seeds by g2pc.synth, so only outputs are stored.

    G2PC_REFERENCE_ROOT=<reference checkout> python tests/golden/make_golden.py          CPU vectors, through
                                                                                         oracle/ref_shim.py
    python tests/golden/make_golden.py --gpu        tiles_ref.npz, tiles_edge.npz: the reference's CUDA rasterizer
                                                    (compiled into oracle/_ref by oracle/build_ref.py), run on an H100
    --edge                                          only the edge-scene vectors (colour_edge.npz, or tiles_edge.npz
                                                    with --gpu)
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "3dgs-to-pc_b200"))

from oracle import philox, ref_shim  # noqa: E402
from g2pc import synth  # noqa: E402

SAMPLING_CASES = {
    # name: (n_gaussians, scene_seed, num_points, exact_num_points, attempts, rng_seed)
    "sampling_a": (1500, 1301, 12000, False, 5, 42),
    "sampling_b": (800, 1302, 9000, True, 100, 43),
}


def make_sampling(name, n, scene_seed, num_points, exact, attempts, rng_seed):
    ref = ref_shim.load()
    sc = synth.make_scene(n, seed=scene_seed)
    eps_fn = lambda g, k, a: philox.draw_eps(g, k, a, rng_seed, 0)
    with ref_shim.cpu_redirect():
        G = ref.gauss_handler.Gaussians(sc["xyz"].clone(), sc["scales"].clone(), sc["rots"].clone(),
                                        sc["colours"].clone() * 255, sc["opacities"].clone())
        G.calculate_normals()
        cov0 = G.covariances.clone()
        keep = G.validate_covariances()
        mags = G.get_gaussian_magnitudes()
        ppg = ref.gauss_to_pc.distribute_points(mags, num_points).type(torch.int)
        with ref_shim.EpsInjector(ref, G.xyz, eps_fn) as inj:
            pts, cols, nrm = ref.gauss_to_pc.generate_pointcloud(
                G, num_points, mahalanobis_distance_std=2.0, exact_num_points=exact,
                num_sample_attempts=attempts, device="cpu", quiet=True)
            calls = np.array([(k, a, len(g)) for (k, a, g) in inj.log], dtype=np.int64)
    np.savez_compressed(
        os.path.join(HERE, name + ".npz"),
        meta=np.array([n, scene_seed, num_points, int(exact), attempts, rng_seed], dtype=np.int64),
        cov0=cov0.numpy(), cov=G.covariances.numpy(), keep=keep.numpy(), normals=G.normals.numpy(),
        magnitudes=mags.numpy(), ppg=ppg.numpy(), points=pts.numpy(), colours=cols.numpy().astype(np.float32),
        point_normals=nrm.numpy().astype(np.float32), mvn_calls=calls)
    print(name, "points", tuple(pts.shape), "mvn calls", calls.shape[0])


COLOUR_CASES = {
    # name: (n_gaussians, scene_seed, n_cameras, colour_resolution)
    "colour_a": (2500, 1310, 2, 200),
    "colour_b": (1200, 1311, 3, 180),
}


def make_colour(name, n, scene_seed, ncams, res):
    """GaussPythonRenderer of the reference (gauss_render.py:210-465), tile parameters pinned to (60, 60000)."""
    ref = ref_shim.load()
    sc = synth.make_scene(n, seed=scene_seed)
    cams, intr = synth.make_cameras(ncams)
    with ref_shim.cpu_redirect(pinned_tiles=(60, 60000)):
        G = ref.gauss_handler.Gaussians(sc["xyz"].clone(), sc["scales"].clone(), sc["rots"].clone(),
                                        sc["colours"].clone(), sc["opacities"].clone())
        R = ref.gauss_render.get_renderer("python", G.xyz, torch.unsqueeze(torch.clone(G.opacities), 1), G.colours,
                                          G.covariances, visible_gaussian_threshold=0.05)
        imgs = []
        for c2w, k in zip(cams, intr):
            cam = ref.camera_handler.get_camera("python", c2w.clone(), k, colour_resolution=res)
            img, _, _, _ = R(cam)
            imgs.append(img.numpy().astype(np.float32))
        np.savez_compressed(os.path.join(HERE, name + ".npz"),
                            meta=np.array([n, scene_seed, ncams, res], dtype=np.int64),
                            max_contribution=R.gaussian_max_contribution.numpy(),
                            colours=R.gaussian_colours.numpy(), images=np.stack(imgs),
                            visible=R.get_visible_gaussians().numpy())
    print(name, "images", np.stack(imgs).shape, "seen", int((R.gaussian_max_contribution > 0).sum()))


def make_sh(name="sh_a", n=400, seed=1320):
    """eval_sh of the reference (gauss_render.py:43-99), degrees 0..3, on seeded coefficients / unit directions; the
    rendered colour is eval_sh + 0.5 clamped at 0 (forward.cu:65-72)."""
    ref = ref_shim.load()
    g = torch.Generator().manual_seed(seed)
    sh = (0.4 * torch.randn(n, 3, 16, generator=g)).float()
    d = torch.randn(n, 3, generator=g)
    d = (d / d.norm(dim=1, keepdim=True)).float()
    out = {f"deg{deg}": ref.gauss_render.eval_sh(deg, sh[..., : (deg + 1) ** 2], d).numpy() for deg in range(4)}
    np.savez_compressed(os.path.join(HERE, name + ".npz"), meta=np.array([n, seed], dtype=np.int64), **out)
    print(name, {k: v.shape for k, v in out.items()})


def _sha(a):
    import hashlib
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest(), dtype=np.uint8)


def make_live_small(name="live_small"):
    """generate_pointcloud of the reference on a 600-Gaussian scene (eps keyed by seed 5): the shape and the SHA-256 of
    the exact bytes of its points and colours (bit-exact comparison without storing the cloud)."""
    ref = ref_shim.load()
    sc = synth.make_scene(600, seed=77)
    eps_fn = lambda g, k, a: philox.draw_eps(g, k, a, 5, 0)
    with ref_shim.cpu_redirect():
        G = ref.gauss_handler.Gaussians(sc["xyz"].clone(), sc["scales"].clone(), sc["rots"].clone(),
                                        sc["colours"].clone() * 255, sc["opacities"].clone())
        G.calculate_normals()
        G.validate_covariances()
        with ref_shim.EpsInjector(ref, G.xyz, eps_fn):
            pts, cols, nrm = ref.gauss_to_pc.generate_pointcloud(G, 5000, device="cpu", quiet=True)
    np.savez_compressed(os.path.join(HERE, name + ".npz"), meta=np.array([600, 77, 5000, 5], dtype=np.int64),
                        points_shape=np.array(pts.shape, dtype=np.int64), points_dtype=np.array(str(pts.dtype)),
                        colours_dtype=np.array(str(cols.dtype)), points_sha256=_sha(pts.numpy()),
                        colours_sha256=_sha(cols.numpy()))
    print(name, "points", tuple(pts.shape), pts.dtype, cols.dtype)


def make_transforms(name="transforms_ref"):
    """load_transform_data of the reference on the transforms.json / COLMAP text / COLMAP binary files that
    tests/test_io_cpu.py writes, skip rates 0 and 2: names, 4x4 matrices and intrinsics."""
    import tempfile
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from test_io_cpu import write_transforms_json, _write_colmap
    ref = ref_shim.load()
    cams, intr = synth.make_cameras(7)
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        for kind in ("json", "colmap_txt", "colmap_bin"):
            if kind == "json":
                path = os.path.join(tmp, "transforms.json")
                write_transforms_json(path, cams, intr)
            else:
                path = os.path.join(tmp, kind)
                _write_colmap(path, cams, binary=(kind == "colmap_bin"))
            for skip in (0, 2):
                tr, ik = ref.transform_dataloader.load_transform_data(path, skip_rate=skip)
                key = f"{kind}_{skip}"
                out[key + "_names"] = np.array(list(tr.keys()))
                out[key + "_matrices"] = np.array([np.asarray(tr[k], dtype=np.float64) for k in tr])
                out[key + "_intrinsics"] = np.array([[float(v) for v in ik[k]] for k in tr], dtype=np.float64)
    np.savez_compressed(os.path.join(HERE, name + ".npz"), **out)
    print(name, sorted(out))


def _edge_scenes():
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import edge_scenes
    return edge_scenes.golden_scenes()


def make_colour_edge(name="colour_edge"):
    """GaussPythonRenderer of the reference on the edge scenes (inside, huge, ties, opacity), tile parameters pinned to
    (60, 60000), every camera at its native size: images, accumulated max contributions and colours per scene."""
    ref = ref_shim.load()
    out = {}
    for key, (sc, cams, intr) in _edge_scenes().items():
        with ref_shim.cpu_redirect(pinned_tiles=(60, 60000)):
            G = ref.gauss_handler.Gaussians(sc["xyz"].clone(), sc["scales"].clone(), sc["rots"].clone(),
                                            sc["colours"].clone(), sc["opacities"].clone())
            R = ref.gauss_render.get_renderer("python", G.xyz, torch.unsqueeze(torch.clone(G.opacities), 1), G.colours,
                                              G.covariances, visible_gaussian_threshold=0.05)
            imgs = []
            for c2w, k in zip(cams, intr):
                cam = ref.camera_handler.get_camera("python", c2w.clone(), k, colour_resolution=int(k[0]))
                img, _, _, _ = R(cam)
                imgs.append(img.numpy().astype(np.float32))
            out[f"{key}_cov"] = G.covariances.numpy()
            out[f"{key}_images"] = np.stack(imgs)
            out[f"{key}_max_contribution"] = R.gaussian_max_contribution.numpy()
            out[f"{key}_colours"] = R.gaussian_colours.numpy()
        print(name, key, out[f"{key}_images"].shape, "seen", int((out[f"{key}_max_contribution"] > 0).sum()))
    np.savez_compressed(os.path.join(HERE, name + ".npz"), **out)


def make_tiles_edge(name="tiles_edge"):
    """The reference's CUDA rasterizer (surface distance on) on the edge scenes, camera matrices from
    oracle.render_cuda.RasterSettings at native size: per camera radii and full colour / depth images, accumulated max /
    total contributions and minimum surface distances per scene."""
    from oracle import gaussians as og, render_cuda as orc
    C = _reference_C()
    dev = "cuda:0"
    out = {}
    for key, (sc, cams, intr) in _edge_scenes().items():
        cov = og.build_covariance(sc["scales"], sc["rots"])
        cov6 = cov.reshape(-1, 9)[:, [0, 1, 2, 4, 5, 8]].float().to(dev)
        xyz, col = sc["xyz"].float().to(dev), sc["colours"].float().to(dev)
        opa = sc["opacities"].float().unsqueeze(1).to(dev)
        n = xyz.shape[0]
        kmax = torch.zeros(n, device=dev)
        ktot = torch.zeros(n, device=dev)
        kdist = torch.full((n,), torch.finfo(torch.float).max, device=dev)
        empty = torch.Tensor([])
        radii, imgs, deps = [], [], []
        for c2w, k in zip(cams, intr):
            rs = orc.RasterSettings(c2w, k)
            H, W = rs.image_height, rs.image_width
            mask = torch.ones(H * W, dtype=torch.int32, device=dev)
            o = C.rasterize_gaussians(torch.as_tensor(rs.bg, device=dev), xyz, col, opa, empty, empty, 1.0, cov6,
                                      rs.viewmatrix.to(dev), rs.projmatrix.to(dev), rs.tanfovx, rs.tanfovy, H, W, empty,
                                      3, rs.campos.to(dev), mask, False, False, True, True)
            _, colour, depth, r, _, _, _, _, contrib, surf, _ = o
            upd = contrib > kmax
            kmax[upd] = contrib[upd]
            ktot += contrib
            kdist = torch.minimum(kdist, surf)
            radii.append(r.cpu().numpy().astype(np.int32))
            imgs.append(colour.cpu().numpy())
            deps.append(depth[0].cpu().numpy())
        out[f"{key}_radii"] = np.stack(radii)
        out[f"{key}_images"] = np.stack(imgs)
        out[f"{key}_depths"] = np.stack(deps)
        out[f"{key}_max_contribution"] = kmax.cpu().numpy()
        out[f"{key}_total_contribution"] = ktot.cpu().numpy()
        out[f"{key}_min_surface_distance"] = kdist.cpu().numpy()
        print(name, key, out[f"{key}_images"].shape, "seen", int((kmax > 0).sum()))
    np.savez_compressed(os.path.join(HERE, name + ".npz"), gpu=np.array(torch.cuda.get_device_name(0)), **out)


TILES_REF = dict(n=8000, scene_seed=1253, ncams=4, res=720, pixels=1024, pixel_seed=7)


def _reference_C():
    """The reference's compiled `_C` from oracle/_ref, loaded on its own (the product ships a package of the same name)."""
    import glob
    import importlib.util
    so = glob.glob(os.path.join(ROOT, "oracle", "_ref", "gaussian_pointcloud_rasterization", "_C*.so"))
    if not so:
        raise SystemExit("oracle/_ref holds no reference extension: run oracle/build_ref.py first")
    spec = importlib.util.spec_from_file_location("g2pc_reference_ext._C", so[0])
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def make_tiles_ref(name="tiles_ref"):
    """The reference's CUDA rasterizer (rasterize_gaussians, surface distance on) over TILES_REF's scene and cameras,
    camera matrices from oracle.render_cuda.RasterSettings, per-camera outputs accumulated as the reference's
    GaussianRasterizer.forward does.  Stored: radii per camera, colour + depth at a seeded sample of pixels per camera,
    the accumulated max / total contributions and the low-surface-distance mask (std 2.0)."""
    from oracle import gaussians as og, render_cuda as orc
    C = _reference_C()
    t = TILES_REF
    dev = "cuda:0"
    sc = synth.make_scene(t["n"], seed=t["scene_seed"], sh_degree=3)
    cov = og.build_covariance(sc["scales"], sc["rots"])
    cov6 = cov.reshape(-1, 9)[:, [0, 1, 2, 4, 5, 8]].float().to(dev)
    xyz, col = sc["xyz"].float().to(dev), sc["colours"].float().to(dev)
    opa = sc["opacities"].float().unsqueeze(1).to(dev)
    n = t["n"]
    kmax = torch.zeros(n, device=dev)
    ktot = torch.zeros(n, device=dev)
    kdist = torch.full((n,), torch.finfo(torch.float).max, device=dev)
    empty = torch.Tensor([])
    cams, intr = synth.make_cameras(t["ncams"])
    radii, img_s, dep_s = [], [], []
    for c2w, k in zip(cams, intr):
        rs = orc.RasterSettings(c2w, k, colour_resolution=t["res"])
        H, W = rs.image_height, rs.image_width
        mask = torch.ones(H * W, dtype=torch.int32, device=dev)
        out = C.rasterize_gaussians(torch.as_tensor(rs.bg, device=dev), xyz, col, opa, empty, empty, 1.0, cov6,
                                    rs.viewmatrix.to(dev), rs.projmatrix.to(dev), rs.tanfovx, rs.tanfovy, H, W, empty, 3,
                                    rs.campos.to(dev), mask, False, False, True, True)
        _, colour, depth, r, _, _, _, _, contrib, surf, _ = out
        upd = contrib > kmax
        kmax[upd] = contrib[upd]
        ktot += contrib
        kdist = torch.minimum(kdist, surf)
        pix = np.random.default_rng(t["pixel_seed"]).choice(H * W, t["pixels"], replace=False)
        p = torch.as_tensor(pix, device=dev)
        radii.append(r.cpu().numpy().astype(np.int16))
        img_s.append(colour.reshape(3, -1)[:, p].cpu().numpy())
        dep_s.append(depth.reshape(-1)[p].cpu().numpy())
    fin = kdist < torch.finfo(torch.float).max
    low = kdist < kdist[fin].mean() * 2.0
    np.savez_compressed(os.path.join(HERE, name + ".npz"), meta=np.array([t[k] for k in TILES_REF], dtype=np.int64),
                        radii=np.stack(radii), image_sample=np.stack(img_s), depth_sample=np.stack(dep_s),
                        max_contribution=kmax.cpu().numpy(), total_contribution=ktot.cpu().numpy(),
                        low_surface=low.cpu().numpy(), gpu=np.array(torch.cuda.get_device_name(0)))
    print(name, "radii", np.stack(radii).shape, "seen", int((kmax > 0).sum()))


if __name__ == "__main__":
    torch.manual_seed(0)
    edge_only = "--edge" in sys.argv  # only the edge-scene vectors (colour_edge, or tiles_edge with --gpu)
    if "--gpu" in sys.argv:
        if not edge_only:
            make_tiles_ref()
        make_tiles_edge()
        raise SystemExit(0)
    if not edge_only:
        make_sh()
        make_live_small()
        make_transforms()
        for name, args in SAMPLING_CASES.items():
            make_sampling(name, *args)
        for name, args in COLOUR_CASES.items():
            make_colour(name, *args)
    make_colour_edge()
