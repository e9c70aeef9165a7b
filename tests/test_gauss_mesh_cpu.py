"""CPU: gauss_to_mesh.py's arguments (defaults, and every refusal raised before any file is opened), gauss_to_pc.py still
refusing --generate_mesh, and the float64 restatement of g2pc_face_cameras on hand cases."""
import numpy as np
import pytest

import f64ref_face_cameras as fo


def _argv(tmp_path, *extra, transforms=True):
    a = ["--input_path", str(tmp_path / "missing.ply")]
    if transforms:
        a += ["--transform_path", str(tmp_path / "missing.json")]
    return a + list(extra)


def test_defaults(tmp_path):
    import gauss_to_mesh
    args = gauss_to_mesh.config_parser(_argv(tmp_path))
    assert args.generate_mesh and args.renderer_type == "cuda"
    assert (args.poisson_depth, args.laplacian_iterations) == (10, 10)
    assert (args.output_path, args.mesh_output_path) == ("3dgs_pc.ply", "3dgs_mesh.ply")
    assert not args.clean_pointcloud and not args.no_prioritise_visible_gaussians
    for d in (2, 10):
        assert gauss_to_mesh.config_parser(_argv(tmp_path, "--poisson_depth", str(d))).poisson_depth == d
    assert gauss_to_mesh.config_parser(_argv(tmp_path, "--laplacian_iterations", "0")).laplacian_iterations == 0


@pytest.mark.parametrize("extra,transforms", [
    (["--renderer_type", "python"], True),
    (["--poisson_depth", "1"], True),
    (["--poisson_depth", "11"], True),
    (["--poisson_depth", "12"], True),
    (["--laplacian_iterations", "-1"], True),
    ([], False),
    (["--no_render_colours"], True),
    (["--no_calculate_normals"], True),
])
def test_refusals_before_loading(tmp_path, extra, transforms):
    """main() with a missing input file: the refusal comes before any loading (else FileNotFoundError or a CUDA error)."""
    import gauss_to_mesh
    with pytest.raises(AttributeError):
        gauss_to_mesh.main(_argv(tmp_path, *extra, transforms=transforms))


def test_gauss_to_pc_still_refuses_generate_mesh(tmp_path):
    import gauss_to_pc as g2p
    with pytest.raises(AttributeError, match="gauss_to_mesh.py"):
        g2p.config_parser(_argv(tmp_path, "--generate_mesh"))
    assert not g2p.config_parser(_argv(tmp_path)).generate_mesh


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_restatement_hand_cases(dtype):
    means, nrm, ids, cam_of, cams, flip, counts = fo.face_camera_hand_cases(dtype)
    out, got = fo.face_cameras(means, nrm, ids, cam_of, cams)
    assert np.array_equal(got, counts) and tuple(counts) == (3, 1, 5, 4)
    assert out.dtype == nrm.dtype
    bits = lambda a: a.view(np.uint32 if a.dtype == np.float32 else np.uint64)
    sign = np.uint32(1 << 31) if dtype == np.float32 else np.uint64(1 << 63)
    assert np.array_equal(bits(out[flip]), bits(nrm[flip]) ^ sign)  # only the sign bits change, zeros included
    assert np.array_equal(bits(out[~flip]), bits(nrm[~flip]))  # everything else is copied, NaN included
    assert np.signbit(out[4]).tolist() == [False, True, False]  # (-0, +0, -1) -> (+0, -0, +1)


def test_restatement_random_rows_face_their_camera():
    rng = np.random.default_rng(3)
    m, N, ncam = 2000, 3000, 7
    cams = rng.normal(size=(ncam, 3)).astype(np.float32) * 5
    ids = rng.choice(N, m, replace=False).astype(np.int32)
    cam_of = rng.integers(0, ncam, N).astype(np.int32)
    means = rng.normal(size=(m, 3)).astype(np.float32)
    nrm = rng.normal(size=(m, 3)).astype(np.float32)
    out, counts = fo.face_cameras(means, nrm, ids, cam_of, cams)
    d = cams[cam_of[ids]].astype(np.float64) - means
    assert (np.einsum("ij,ij->i", out.astype(np.float64), d) > 0).all() and counts[1:].sum() == 0
    out2, counts2 = fo.face_cameras(means, -nrm, ids, cam_of, cams)
    assert np.array_equal(out2, out) and counts2[0] == m - counts[0]
