"""`EnvSpinDecorator` (ca_code/utils/light_decorator.py:18-164) with the lighting built on the GPU
(csrc/envmap_prefilter.cu):

* construction: the probe is read on the host with cv2 as the reference does (imread, ydown flip, INTER_AREA resize to
  1024x512) and its 90th percentile taken with numpy; everything after that runs on the device.  The mip chain is the
  raw probe at level 0 and, at levels i >= 1, the area-halved sin-weighted probe prefiltered at sigma = i * sigma_step
  with 4096 samples, all levels in one launch of `gb_envmap_prefilter_sg`.
* every frame: `gb_envmap_spin_table` writes lightrot, envbg, the 16x32 light table (envmap, light_intensity) and the
  normalisation for the whole batch without a host synchronisation or copy; the mip chain scaled by
  2 pi norm_scale[0] (the reference's quirk: item 0's scale for the whole batch) and the constant light positions are
  torch ops on device tensors.  With a fixed batch size the frame can be captured in a CUDA graph.

The dict handed to `mod` has the reference's keys, shapes and dtypes.

`SingleLightCycleDecorator` (light_decorator.py:167-218) is host-side, as in the reference: one unit point light per
item on a circle of radius 1100 around the head, read from the head translation on the host."""
import ctypes

import cv2
import numpy as np
import torch as th
import torch.nn.functional as thf

from . import _lib
from .envmap import _prefilter_levels

NUM_SAMPLES = 4096        # light_decorator.py:69
PROBE_HW = (512, 1024)    # cv2.resize(image, (1024, 512)), light_decorator.py:58
MAX_MIPLEVEL = 8          # levels the environment-map specular kernel takes


def _sph_grid(height, width, device):
    """the unit direction of each texel centre of a height x width latitude-longitude map [1,3,H,W]
    (light_decorator.py:75-90)"""
    theta, phi = th.meshgrid(
        (th.arange(height, dtype=th.float32, device=device) + 0.5) * np.pi / height,
        (th.arange(-width // 2, width // 2, dtype=th.float32, device=device) + 0.5) * np.pi * 2 / width,
        indexing="ij")
    return th.stack([th.sin(theta) * th.sin(phi), th.cos(theta), -th.sin(theta) * th.cos(phi)], dim=0)[None]


class EnvSpinDecorator(th.nn.Module):
    def __init__(self, mod, envmap_path, envmap_dist=10000.0, env_scale=18.0, cycle=256, sigma_step=0.2, miplevel=4,
                 ydown=False):
        """envmap_path: an HDR file cv2 reads, or the H x W x 3 array cv2.imread(path, -1) would return (BGR)."""
        super().__init__()
        if not isinstance(miplevel, int) or not 1 <= miplevel <= MAX_MIPLEVEL:
            raise ValueError("EnvSpinDecorator: miplevel must be an int in 1..%d (got %r)" % (MAX_MIPLEVEL, miplevel))
        if miplevel > 1 and not sigma_step > 0:
            raise ValueError("EnvSpinDecorator: sigma_step must be > 0 (got %r)" % (sigma_step,))
        if not cycle:
            raise ValueError("EnvSpinDecorator: cycle must be non-zero")
        self.mod = mod
        self.envmap_dist = envmap_dist
        self.env_scale = env_scale
        self.cycle = cycle
        self.sigma_step = sigma_step
        self.miplevel = miplevel
        self.ydown = ydown

        probe = self._read_probe(envmap_path)
        # np.percentile of the static probe, once (the reference recomputes it for every item of every frame)
        self.perc90 = float(np.percentile(probe, 90))
        if not self.perc90 > 0:
            raise ValueError("EnvSpinDecorator: the probe's 90th percentile must be positive (got %r)" % self.perc90)
        self._set_lightmap(probe)

        L = 16
        theta, phi = np.meshgrid((np.arange(L, dtype=np.float32) + 0.5) * np.pi / L,
                                 (np.arange(-L, L, dtype=np.float32) + 0.5) * np.pi / L, indexing="ij")
        sph = np.stack([np.sin(theta) * np.sin(phi), np.cos(theta), -np.sin(theta) * np.cos(phi)], axis=0).reshape((3, -1))
        self.register_buffer("sphvec", th.from_numpy(sph).to(self.image.device))

    def _read_probe(self, envmap_path):
        """[3,512,1024] float32 numpy, read and resized as light_decorator.py:55-62 does"""
        image = envmap_path if isinstance(envmap_path, np.ndarray) else cv2.imread(envmap_path, -1)
        if image is None:
            raise ValueError("EnvSpinDecorator: cannot read %r" % (envmap_path,))
        if image.ndim != 3 or image.shape[2] != 3 or image.shape[0] < 1 or image.shape[1] < 1:
            raise ValueError("EnvSpinDecorator: the probe must be H x W x 3 (got %s)" % (image.shape,))
        image = image[:, :, ::-1]
        if self.ydown:
            image = image[::-1, ::-1]
        image = cv2.resize(image, PROBE_HW[::-1], interpolation=cv2.INTER_AREA)
        return np.ascontiguousarray(np.ascontiguousarray(image).astype(np.float32).transpose(2, 0, 1))

    def _set_lightmap(self, probe):
        dev = th.device("cuda", th.cuda.current_device())
        # the probe stays a device buffer outside the state dict (the reference keeps it as a plain attribute)
        self.register_buffer("image", th.from_numpy(probe).to(dev), persistent=False)
        H = self.image.shape[1]
        multisin = th.sin((th.arange(H, device=dev) + 0.5) * np.pi / H)[None, None, :, None]
        mipmap = [self.image[None].clone()]
        image = self.image[None].clone() * multisin
        levels = []
        for i in range(self.miplevel - 1):
            image = thf.interpolate(image, None, scale_factor=0.5, mode="area")
            levels.append(((i + 1) * self.sigma_step, _sph_grid(image.shape[2], image.shape[3], dev), image, None))
        if levels:
            mipmap += _prefilter_levels(levels, NUM_SAMPLES)
        for i, p in enumerate(mipmap):
            self.register_buffer(f"mipmap_{i}", p)

    def mipmap(self, bsize, device, scale=1.0):
        return [getattr(self, f"mipmap_{i}").expand(bsize, -1, -1, -1).to(device) * scale for i in range(self.miplevel)]

    def light_table(self, index, batch_size):
        """lightrot [B,3,3], envbg [B,3,512,1024] (already / 255), envmap [B,3,16,32], light_intensity [B,512,3],
        norm_scale [B] for the rotation angles 2 pi index / cycle.  `index` is read on the host (a list, a numpy array
        or a CPU tensor; a CUDA tensor costs a synchronisation)."""
        index = index.tolist() if th.is_tensor(index) else list(index)
        if len(index) < batch_size:
            raise ValueError("EnvSpinDecorator: %d indices for a batch of %d" % (len(index), batch_size))
        B = batch_size
        img = self.image
        _lib.check_input(img, "image")
        He, We = img.shape[1:]
        f32 = dict(device=img.device, dtype=th.float32)
        lightrot = th.empty(B, 3, 3, **f32)
        envbg = th.empty(B, 3, He, We, **f32)
        hpass = th.empty(B, 3, He, 32, **f32)
        envmap = th.empty(B, 3, 16, 32, **f32)
        light_intensity = th.empty(B, 512, 3, **f32)
        norm_scale = th.empty(B, **f32)
        angles = (ctypes.c_float * B)(*[2.0 * np.pi * float(index[i]) / self.cycle for i in range(B)])
        with th.cuda.device(img.device):
            _lib.check(_lib.lib().gb_envmap_spin_table(
                B, He, We, angles, _lib.ptr(img), self.perc90, float(self.env_scale), _lib.ptr(lightrot),
                _lib.ptr(envbg), _lib.ptr(hpass), _lib.ptr(envmap), _lib.ptr(light_intensity), _lib.ptr(norm_scale),
                _lib.stream_ptr(img.device)), "envmap_spin_table")
        return lightrot, envbg, envmap, light_intensity, norm_scale

    def forward(self, **data):
        device = data["campos"].device
        batch_size = data["campos"].size(0)
        lightrot, envbg, envmaps, light_intensity, norm_scale = self.light_table(data["index"], batch_size)
        light_dir = self.sphvec.view(3, -1).t()[None].expand(batch_size, -1, -1).contiguous()

        data["preconv_envmap"] = self.mipmap(batch_size, device, 2.0 * np.pi * norm_scale[0])
        data["sigma_step"] = self.sigma_step
        data["envmap"] = envmaps.to(device)
        data["lightrot"] = lightrot.to(device)
        data["light_intensity"] = light_intensity.to(device)
        data["light_pos"] = self.envmap_dist * light_dir.to(device)
        data["envbg"] = envbg.to(device)
        data["light_type"] = "envmap"
        data["n_lights"] = light_intensity.shape[1] * th.ones(batch_size, 1, device=device)
        data["is_fullylit_frame"] = th.zeros(1, device=device)
        return self.mod(**data)


def single_light_position(index, cycle, light_rotate_axis, trans=None):
    """light_decorator.py:185-208: the float32 [3] light position of frame `index` on a circle of radius 1100 about
    axis 0 (the y-z plane), 1 (x-z at height 300, then rescaled to 1100) or any other value (x-y), plus `trans`"""
    index = index % cycle
    angle = (abs(index) / cycle) * 2 * np.pi
    if light_rotate_axis == 0:
        lpos = np.asarray([0.0, 1100.0 * np.sin(angle), 1100.0 * np.cos(angle)]).astype(np.float32)
    elif light_rotate_axis == 1:
        lpos = np.asarray([-1.0 * 1100.0 * np.sin(angle), 300.0, 1100.0 * np.cos(angle)]).astype(np.float32)
    else:
        lpos = np.asarray([1100.0 * np.cos(angle), 1100.0 * np.sin(angle), 0.0]).astype(np.float32)
    lpos = 1100.0 * lpos / np.linalg.norm(lpos)
    if trans is not None:
        lpos += trans
    return lpos


class SingleLightCycleDecorator(th.nn.Module):
    """Sets one unit-intensity point light per item, cycling with data["index"] (cycle frames per turn), and
    n_lights = 1: light_intensity [B,1,1], light_pos [B,1,3] (head_pose[:, :3, 3] or pose[:, :3] added, read on the
    host), n_lights [B] int32, is_fullylit_frame [1]."""

    def __init__(self, mod: th.nn.Module, cycle: int = 256, light_rotate_axis: int = 0) -> None:
        super().__init__()
        self.mod = mod
        self.cycle = cycle
        self.light_rotate_axis = light_rotate_axis

    def forward(self, **data):
        device = data["campos"].device
        batch_size = data["campos"].size(0)
        trans = None
        if "head_pose" in data:
            trans = data["head_pose"][:, :3, 3].detach().cpu().numpy()
        elif "pose" in data:
            trans = data["pose"][:, :3].detach().cpu().numpy()
        index = data["index"]
        index = index.tolist() if th.is_tensor(index) else list(index)
        pos = np.stack([single_light_position(index[i], self.cycle, self.light_rotate_axis,
                                              None if trans is None else trans[i]) for i in range(batch_size)])
        data["light_intensity"] = th.ones(batch_size, 1, 1, device=device)
        data["light_pos"] = th.from_numpy(pos).float().to(device)[:, None]
        data["n_lights"] = th.ones(batch_size, device=device).int()
        data["is_fullylit_frame"] = th.zeros(1, device=device)
        return self.mod(**data)
