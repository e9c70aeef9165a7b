"""Camera model — drop-in for the reference's camera_handler.py (same names and signatures).

Reference: camera_handler.py (fov/focal helpers :8-12, getProjectionMatrix :14-34, Camera :36-50,
get_camera :53-108).  The 4x4 matrix algebra is tiny host-side set-up (one camera per call) and stays in torch; the
matrices are handed to the colour kernels by value (g2pc_camera_t).
"""
import math

import torch


def fov2focal(fov, pixels):
    return pixels / (2 * math.tan(fov / 2))


def focal2fov(focal, pixels):
    return 2 * math.atan(pixels / (2 * focal))


def getProjectionMatrix(znear, zfar, fovX, fovY):
    """Perspective matrix of the reference (camera_handler.py:14-34): symmetric frustum, +z convention, so that
    w_clip = z_view.  Only five entries are non-zero."""
    half_w = math.tan(fovX / 2) * znear
    half_h = math.tan(fovY / 2) * znear
    depth = zfar - znear
    return torch.tensor([[znear / half_w, 0.0, 0.0, 0.0],
                         [0.0, znear / half_h, 0.0, 0.0],
                         [0.0, 0.0, zfar / depth, -(zfar * znear) / depth],
                         [0.0, 0.0, 1.0, 0.0]], dtype=torch.float32)


class Camera():
    """Pinhole camera of the python renderer (camera_handler.py:36-50): OpenGL c2w (looks down -z), row-vector
    view matrix world_view_transform = inv(c2w)^T, znear 10, zfar 100.

    The 4x4 algebra runs on the host in float32 (the kernels take the matrices by value); the tensor attributes of the
    reference (world_view_transform, projection_matrix, camera_center, full_proj_transform) are exposed on c2w's
    device on first access."""

    def __init__(self, width, height, focal_x, focal_y, c2w, znear=10, zfar=100):
        self.znear = znear
        self.zfar = zfar
        self.focal_x = focal_x
        self.focal_y = focal_y
        self.FoVx = focal2fov(self.focal_x, width)
        self.FoVy = focal2fov(self.focal_y, height)
        self.image_width = int(width)
        self.image_height = int(height)
        self.c2w = c2w
        host = c2w.detach().to("cpu", torch.float32)
        self._host = {}
        self._host["world_view_transform"] = torch.linalg.inv(host).permute(1, 0).contiguous()
        self._host["projection_matrix"] = getProjectionMatrix(znear=self.znear, zfar=self.zfar, fovX=self.FoVx,
                                                               fovY=self.FoVy).transpose(0, 1).contiguous()
        self._host["camera_center"] = self._host["world_view_transform"].inverse()[3, :3].contiguous()
        self._host["full_proj_transform"] = self._host["world_view_transform"] @ self._host["projection_matrix"]
        self._dev = {}

    def host(self, name):
        return self._host[name]

    def __getattr__(self, name):
        h = self.__dict__.get("_host", {})
        if name in h:
            d = self.__dict__["_dev"]
            if name not in d:
                d[name] = h[name].to(self.__dict__["c2w"].device)
            return d[name]
        raise AttributeError(name)


def get_camera(renderer_type, transform, cam_intrinsic, colour_resolution=None, sh_degree=3, white_bkgd=True, mask=None):
    """Per-camera object for `renderer(camera)` (camera_handler.py:53-108).

    cam_intrinsic = [w, h, fx, fy].  Without a mask the image is rescaled to `colour_resolution` pixels wide (focal
    lengths scale along); with a mask the native size is kept and the mask must match it (it is returned flattened on
    the camera as `.mask`)."""
    native_w, native_h = int(cam_intrinsic[0]), int(cam_intrinsic[1])
    scale = 1 if (colour_resolution is None or mask is not None) else colour_resolution / native_w
    if mask is not None:
        if tuple(mask.shape[:2]) != (native_h, native_w):
            raise Exception("Size of mask must match size of input image")
        mask = mask.flatten()
    if renderer_type == "cuda":
        return _cuda_settings(transform, int(native_w * scale), int(native_h * scale), float(cam_intrinsic[2]) * scale,
                              float(cam_intrinsic[3]) * scale, sh_degree, white_bkgd, mask)
    if renderer_type != "python":
        raise Exception(f"Renderer of type {renderer_type} is not supported")
    cam = Camera(int(native_w * scale), int(native_h * scale), float(cam_intrinsic[2]) * scale,
                 float(cam_intrinsic[3]) * scale, transform)
    cam.sh_degree = sh_degree
    cam.white_bkgd = white_bkgd
    cam.mask = mask
    return cam


def _cuda_settings(transform, img_width, img_height, focal_x, focal_y, sh_degree, white_bkgd, mask):
    """GaussianRasterizationSettings of the CUDA back-end (camera_handler.py:72-108): the OpenGL c2w is turned into a
    z-forward camera by negating columns 1:3 (the reference does that IN PLACE on the caller's tensor, :75; a copy is
    flipped here), viewmatrix = inv(c2w)^T, projmatrix = viewmatrix @ projection^T, znear 10 / zfar 100, debug=True,
    antialiasing=False.  The 4x4 algebra runs on the host in float32; the settings carry host copies of the matrices
    (the kernels take them by value) next to the tensor fields of the reference."""
    from g2pc.rasterizer import GaussianRasterizationSettings

    class Settings(GaussianRasterizationSettings):
        pass

    dev = transform.device if torch.is_tensor(transform) else torch.device("cpu")
    c2w = torch.as_tensor(transform).detach().to("cpu", torch.float32).clone()
    c2w[:, 1:3] = -c2w[:, 1:3]
    fovX, fovY = focal2fov(focal_x, img_width), focal2fov(focal_y, img_height)
    proj = getProjectionMatrix(znear=10, zfar=100, fovX=fovX, fovY=fovY).transpose(0, 1)
    view = torch.linalg.inv(c2w).permute(1, 0).contiguous()
    campos = view.inverse()[3, :3].contiguous()
    full = (view @ proj).contiguous()
    bg = [1.0, 1.0, 1.0] if white_bkgd else [0.0, 0.0, 0.0]
    on_dev = (lambda t: t.to(dev)) if dev.type == "cuda" else (lambda t: t)
    s = Settings(image_height=int(img_height), image_width=int(img_width), tanfovx=math.tan(fovX * 0.5),
                 tanfovy=math.tan(fovY * 0.5), bg=on_dev(torch.tensor(bg)), scale_modifier=1.0, viewmatrix=on_dev(view),
                 projmatrix=on_dev(full), sh_degree=sh_degree, campos=on_dev(campos), mask=mask, prefiltered=False,
                 debug=True, antialiasing=False)
    s._viewmatrix_host = view.reshape(-1).tolist()
    s._projmatrix_host = full.reshape(-1).tolist()
    s._campos_host = campos.tolist()
    s._bg_host = bg
    return s
