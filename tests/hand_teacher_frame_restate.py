"""Seeded inputs of the relightable hand teacher's frame (`hand_teacher.AutoEncoder`), shared by
tests/golden/make_hand_teacher_frame_golden.py, the CPU and GPU tests and scripts/profile_hand_teacher_frame.py.

The model is the hand frame's (tests/hand_frame_restate.py: assets, configuration, `seeded_fill`) at the example
configuration's size: uv 1024, 4096 primitives of 16 x 16 x 8.  `reduce` applies the fixture's two changes, to the
reference's model and to ours alike: a 128^2 shadow image (the non-persistent `relightdecoder.pixel_coords` buffer,
from which both implementations read the size) and chunks of 1 light, so the fixture's L = 2 lights take two chunks.
The reference's fp64 U-Net at 1024^2 keeps every light's activations for the backward and its convolutions unfold
each item's input: two items per chunk and two lights is what fits in the memory of a 64 GB host."""
import numpy as np
import torch

import hand_frame_restate as hf

SHADOW = 128                  # shadow image side of the fixture (the model's is 1024)
CHUNK = 1                     # relightdecoder.chunksize of the fixture (the model's is 5)
L = 2                         # point lights of the fixture
ENV_H, ENV_W = 200, 208       # env mode render: compose_envmap's mirror ball needs at least 200 x 200
ENVBG_HW = (64, 128)          # env mode background probe
MODES = ("eval", "train0", "train", "fresh", "env")
ITERATION = {"eval": None, "train0": 0, "train": 5000, "fresh": 0, "env": None}
GRAD_MODES = ("train0", "train", "fresh")
PRE_MODULES = ("poseencoder", "poseencoder2", "geomdecoder.transdecoder", "geomdecoder.alphadecoder",
               "relightdecoder")
PRIM_KEYS = ("primpos", "primrot", "primscale", "primrgba", "texolat")


def pixel_coords(size=SHADOW, dtype=torch.float32):
    """the decoder's shadow-image grid, stack([y, x]) as both implementations build it"""
    y, x = torch.meshgrid(torch.arange(size), torch.arange(size), indexing="ij")
    return torch.stack([y, x], dim=-1).to(dtype)


def reduce(model, shadow=SHADOW, chunk=CHUNK):
    dec = model.relightdecoder
    dec.pixel_coords = pixel_coords(shadow).to(dec.pixel_coords.device)
    dec.chunksize = chunk
    return model


def env_config():
    """the env mode's model: no calibration, no blur, a render the mirror ball fits in"""
    c = hf.config(ENV_H, ENV_W)
    c.pop("cal")
    c["learn_blur"] = False
    return c


def lights(points, n=L, batch=2, seed=11):
    """light_pos [B,n,3] at distance 1100 from each item's centroid, light_intensity [B,n,3] in [0.5, 1.5)"""
    g = torch.Generator().manual_seed(seed)
    d = torch.nn.functional.normalize(torch.randn(batch, n, 3, generator=g, dtype=torch.float64), dim=-1)
    pos = points.mean(1)[:, None].double() + 1100.0 * d
    return pos.float(), (0.5 + torch.rand(batch, n, 3, generator=g, dtype=torch.float64)).float()


def envbg(batch=2, seed=13):
    """a smooth [B,3,64,128] environment in 0.2 .. 1.2 (already / 255, as EnvSpinDecorator's)"""
    rng = np.random.default_rng(seed)
    He, We = ENVBG_HW
    y, x = np.mgrid[0:He, 0:We].astype(np.float64)
    out = np.zeros((batch, 3, He, We))
    for b in range(batch):
        for c in range(3):
            for _ in range(3):
                fy, fx = rng.uniform(0.3, 1.5, 2) * 2 * np.pi / np.array([He, We])
                out[b, c] += rng.uniform(0.2, 1.0) * np.sin(fy * y + fx * x + rng.uniform(0, 2 * np.pi))
    lo, hi = out.min(), out.max()
    return torch.from_numpy(0.2 + (out - lo) / (hi - lo)).float()


def grad_param_names(model):
    """the first and last parameter (by name) of each decoder module"""
    names = sorted(n for n, _ in model.named_parameters())
    out = []
    for m in PRE_MODULES:
        sub = [n for n in names if n.startswith(m + ".")]
        out += sorted({sub[0], sub[-1]})
    return out


def functional_weights(shapes, seed=31):
    """the seeded linear functional on the per-primitive outputs and texolat: one fp64 N(0,1) weight per element"""
    g = torch.Generator().manual_seed(seed)
    return {k: torch.randn(shapes[k], generator=g, dtype=torch.float64) for k in PRIM_KEYS if k in shapes}
