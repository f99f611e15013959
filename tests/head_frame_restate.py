"""Seeded assets, configuration, parameters and inputs of the head avatar's frame (`rgca.AutoEncoder`), shared by
tests/golden/make_head_frame_golden.py, the CPU and GPU tests and scripts/profile_head_frame.py, and an fp64 torch
restatement of the frame's light work (rgca.py:175-193 over sh.dir2sh).

The mesh is a bumped, UV-gridded sheet of (N + 1)^2 vertices; its UV index / barycentric images are rasterised here
at the slab's size and given as assets (this project does not rasterise them)."""
import math

import numpy as np
import torch
import torch.nn.functional as F

CAMERAS = ["401033", "400870", "410244", "402100"]   # unsorted on purpose: CalV5 sorts, LearnableBlur does not
IDENTITY = "400870"
BATCH_CAMERAS = ["410244", "401033"]                 # a grey ("41...") and a colour camera
H, W = 208, 256                                      # render size of the tests (compose_envmap needs >= 200)
SLAB = 128                                           # decoder slab of the tests (1024 upstream)
N_LIGHTS = 460                                       # the capture rig's light table


class Assets(dict):
    """the reference's asset object: attribute access and `"key" in assets`"""

    __getattr__ = dict.__getitem__


def sheet(n=16, size=SLAB, seed=11):
    """vi / vti [2 n^2, 3], vt [(n+1)^2, 2], v [(n+1)^2, 3] (mm, a bump of +-200 x +-200 x 60) and the UV images
    index_image / bary_image [size,size,3], face_index_image [size,size], valid_mask [size,size,1]; texels outside
    the central 90 % of the UV square are uncovered (index -1)"""
    g = np.random.default_rng(seed)
    u, v = np.meshgrid(np.linspace(0.0, 1.0, n + 1), np.linspace(0.0, 1.0, n + 1), indexing="xy")
    vt = np.stack([u, v], -1).reshape(-1, 2).astype(np.float32)
    x, y = 400.0 * (u - 0.5), 400.0 * (v - 0.5)
    z = -60.0 * np.exp(-(x ** 2 + y ** 2) / (2 * 120.0 ** 2)) + g.normal(0.0, 2.0, x.shape)
    verts = np.stack([x, y, z], -1).reshape(-1, 3).astype(np.float32)
    tri = []
    for i in range(n):
        for j in range(n):
            a, b, c, d = i * (n + 1) + j, i * (n + 1) + j + 1, (i + 1) * (n + 1) + j, (i + 1) * (n + 1) + j + 1
            tri += [(a, b, d), (a, d, c)]
    vi = np.asarray(tri, np.int64)
    # texel centres; flip_uv: image row 0 is v = 1
    tu, tv = np.meshgrid((np.arange(size) + 0.5) / size, 1.0 - (np.arange(size) + 0.5) / size, indexing="xy")
    cu, cv = tu * n, tv * n
    ci, cj = np.minimum(cv.astype(np.int64), n - 1), np.minimum(cu.astype(np.int64), n - 1)
    fu, fv = cu - cj, cv - ci
    upper = fu >= fv                                  # (a, b, d) where the u-fraction exceeds the v-fraction
    face = 2 * (ci * n + cj) + (~upper)
    w_a = np.where(upper, 1.0 - fu, 1.0 - fv)
    w_b = np.where(upper, fu - fv, fv - fu)
    w_d = np.where(upper, fv, fu)
    bary = np.stack([w_a, w_b, w_d], -1).astype(np.float32)
    index = vi[face]
    valid = (tu > 0.05) & (tu < 0.95) & (tv > 0.05) & (tv < 0.95)
    index[~valid] = -1
    face = np.where(valid, face, -1)
    bary[~valid] = 0.0
    return dict(vi=vi, vti=vi.copy(), vt=vt, v=verts, index_image=index.astype(np.int64), bary_image=bary,
                face_index_image=face.astype(np.int64), valid_mask=valid[..., None])


def assets(slab=SLAB, drop=()):
    """the head's assets with the UV images at slab x slab; `drop` removes UV images by name"""
    s = sheet(size=slab)
    g = np.random.default_rng(5)
    topo = Assets(vi=s["vi"], vt=s["vt"], vti=s["vti"], v=s["v"])
    a = Assets(topology=topo, verts_mean=s["v"], verts_var=float(25.0 ** 2),
               color_mean=torch.from_numpy((255.0 * g.uniform(0.2, 0.8, (3, slab, slab))).astype(np.float32)),
               camera_ids=CAMERAS,
               index_image=s["index_image"], bary_image=s["bary_image"], face_index_image=s["face_index_image"],
               valid_mask=s["valid_mask"])
    for k in drop:
        del a[k]
    return a


def config(h=H, w=W, slab=SLAB):
    """rgca_example.yml's model section at the given render size and decoder slab"""
    dec = {"n_color_sh": 3}
    if slab != 1024:
        dec["slabsize"] = slab
    return {"n_embs": 256, "image_height": h, "image_width": w,
            "encoder": {"noise_std": 1.0, "mean_scale": 0.1, "logvar_scale": 0.01},
            "decoder": dec, "cal": {"identity_camera": IDENTITY}, "learn_blur": True}


def seeded_fill(model, seed=2026):
    """every parameter refilled from a generator seeded by its rank in the sorted names, so the fill does not depend
    on the order in which modules register parameters: weight_v ~ N(0, 1 / fan_in) (fan_in = numel of one row),
    weight_g = ||weight_v|| U(0.8, 1.2), albedo ~ U(0.2, 0.6), the calibration rows (1, 1, 1, 0, 0, 0) + N(0, 0.05^2),
    the blur logits 1 + N(0, 0.3^2), every other parameter (biases) ~ N(0, 0.05^2)"""
    params = dict(model.named_parameters())
    names = sorted(params)
    with torch.no_grad():
        for i, name in enumerate(names):
            p, g = params[name], torch.Generator().manual_seed(seed + i)
            if name.endswith("weight_g"):
                continue
            if name.endswith("weight_v") or name.endswith(".weight"):
                p.copy_(torch.randn(p.shape, generator=g) / math.sqrt(max(p[0].numel(), 1)))
            elif name.endswith("albedo"):
                p.copy_(0.2 + 0.4 * torch.rand(p.shape, generator=g))
            elif name.endswith("holder.params"):
                p.copy_(torch.tensor([1.0, 1.0, 1.0, 0.0, 0.0, 0.0]) + 0.05 * torch.randn(p.shape, generator=g))
            elif name.endswith("weights_raw"):
                p.copy_(1.0 + 0.3 * torch.randn(p.shape, generator=g))
            else:
                p.copy_(0.05 * torch.randn(p.shape, generator=g))
        for i, name in enumerate(names):
            if name.endswith("weight_g"):
                g = torch.Generator().manual_seed(seed + i)
                params[name].copy_(params[name[:-1] + "v"].norm() * (0.8 + 0.4 * torch.rand(params[name].shape,
                                                                                             generator=g)))


def rotation(axis, angle):
    a = torch.as_tensor(axis, dtype=torch.float64)
    a = a / a.norm()
    Kx = torch.tensor([[0.0, -a[2], a[1]], [a[2], 0.0, -a[0]], [-a[1], a[0], 0.0]], dtype=torch.float64)
    return torch.eye(3, dtype=torch.float64) + math.sin(angle) * Kx + (1 - math.cos(angle)) * (Kx @ Kx)


def inputs(batch=2, n_lights=N_LIGHTS, n_active=(300, 460), C=1, h=H, w=W, slab=SLAB, seed=31):
    """the frame's inputs (fp32, CPU): a slightly rotated and translated head, cameras at ~1000 mm looking at it,
    `n_lights` rig lights zero-padded past n_active[b], light_intensity [B,L,C]"""
    g = torch.Generator().manual_seed(seed)
    s = sheet(size=slab)
    hp, Rt, K, campos = [], [], [], []
    for b in range(batch):
        R = rotation([0.2, 1.0, 0.1], 0.15 * (b + 1))
        t = torch.tensor([5.0 * b, -10.0, 20.0], dtype=torch.float64)
        hp.append(torch.cat([R, t[:, None]], 1))
        Rc = rotation([0.0, 1.0, 0.0], math.pi + 0.1 * (b - 0.5))        # camera z axis towards the head's -z side
        cam = -Rc.T @ torch.tensor([0.0, 0.0, 1000.0], dtype=torch.float64)
        Rt.append(torch.cat([Rc, (-Rc @ cam)[:, None]], 1))
        campos.append(cam)
        f = 1.6 * w
        K.append(torch.tensor([[f, 0.0, w / 2.0 + b], [0.0, f * 1.01, h / 2.0 - b], [0.0, 0.0, 1.0]],
                              dtype=torch.float64))
    d = torch.randn(batch, n_lights, 3, generator=g, dtype=torch.float64)
    light_pos = 1100.0 * d / d.norm(dim=-1, keepdim=True)
    intensity = 0.5 + torch.rand(batch, n_lights, C, generator=g, dtype=torch.float64)
    for b in range(batch):
        intensity[b, n_active[b % len(n_active)]:] = 0.0
        light_pos[b, n_active[b % len(n_active)]:] = 0.0
    head_pose = torch.stack(hp)
    light_pos[0, 1] = head_pose[0, :, 3]                 # a light at the head centre
    verts = torch.as_tensor(s["v"], dtype=torch.float64)[None] + torch.randn(batch, s["v"].shape[0], 3, generator=g,
                                                                              dtype=torch.float64)
    color = 255.0 * torch.rand(batch, 3, 1024, 1024, generator=g)
    f32 = lambda t: t.to(torch.float32).contiguous()
    return {"head_pose": f32(head_pose), "campos": f32(torch.stack(campos)), "registration_vertices": f32(verts),
            "color": color, "light_intensity": f32(intensity), "light_pos": f32(light_pos),
            "n_lights": torch.tensor([n_active[b % len(n_active)] for b in range(batch)], dtype=torch.int32),
            "K": f32(torch.stack(K)), "Rt": f32(torch.stack(Rt)), "camera_id": list(BATCH_CAMERAS[:batch])}


def dir2sh64(deg, dirs):
    """sh.dir2sh's basis in fp64, one coefficient at a time from the associated Legendre recurrence in the degree"""
    x, y, z = dirs[..., 0], dirs[..., 1], dirs[..., 2].clamp(-1.0, 1.0)
    ct = torch.cos(torch.acos(z))
    st = torch.sqrt(((1.0 + ct) * (1.0 - ct)).clamp(min=1e-8))
    phi = torch.atan2(y, x)
    out = [None] * ((deg + 1) ** 2)
    for n in range(deg + 1):
        for m in range(-n, n + 1):
            am = abs(m)
            pmm = torch.ones_like(ct)
            for i in range(1, am + 1):
                pmm = -pmm * (2 * i - 1) * st
            if n == am:
                p = pmm
            else:
                p_prev, p = pmm, ct * (2 * am + 1) * pmm
                for i in range(am + 2, n + 1):
                    p_prev, p = p, (ct * (2 * i - 1) * p - (i + am - 1) * p_prev) / (i - am)
            r = 1.0
            for i in range(n - am + 1, n + am + 1):
                r *= i
            k = math.sqrt((2 * n + 1) / (4.0 * math.pi) / r)
            if m > 0:
                out[n * n + n + m] = math.sqrt(2.0) * k * torch.cos(m * phi) * p
            elif m < 0:
                out[n * n + n + m] = math.sqrt(2.0) * k * torch.sin(am * phi) * p
            else:
                out[n * n + n] = k * p
    return torch.stack(out, -1)


def head_lights64(head_pose, campos, Rt, light_pos, light_intensity, lightrot=None, with_terms=False):
    """rgca.py:175-193 restated in fp64; with_terms also returns sum over L of |sh * intensity| [B,3,81]"""
    d = lambda t: t.to(torch.float64)
    head_pose, campos, Rt, light_pos, light_intensity = map(d, (head_pose, campos, Rt, light_pos, light_intensity))
    light_intensity = light_intensity.expand(-1, -1, 3)
    hp4 = torch.cat([head_pose, torch.zeros_like(head_pose[:, :1, :])], 1)
    hp4[:, 3, 3] = 1.0
    R, t = head_pose[:, :3, :3], head_pose[:, :3, 3]
    out = {"headrel_Rt": Rt @ hp4, "headrel_campos": ((campos - t)[:, None] @ R)[:, 0],
           "headrel_light_pos": (light_pos - t[:, None]) @ R}
    sh = dir2sh64(8, F.normalize(out["headrel_light_pos"], p=2, dim=-1))
    terms = sh[:, :, None] * light_intensity[..., None]
    out["headrel_light_sh"] = terms.sum(1)
    out["lightrot"] = None if lightrot is None else d(lightrot) @ R
    if with_terms:
        out["terms_abs"] = terms.abs().sum(1)
    return out


# ----------------------------------------------------------------------------------------- frame fixture helpers
MODES = ("point", "train", "envmap")
PRIM_KEYS = ("primpos", "primqvec", "primscale", "opacity", "diff_color", "spec_color")  # the pre-render functional
RANDOM_KEYS = ("color_rand", "cos_weight")     # drawn with th.rand inside PrimDecoder: shape and finiteness only
SUBMODULES = ("encoder", "geomdecoder", "decoder")


def mode_inputs(mode, batch=2):
    """the frame's keyword arguments (fp32, CPU) for one fixture mode: eval with L = 460 zero-padded point lights;
    training with a background and is_fully_lit_frame = [True, False]; eval environment map (preconv_envmap, envbg,
    lightrot, 512 lights with C = 3)"""
    if mode == "envmap":
        inp = inputs(batch=batch, n_lights=512, n_active=(512,), C=3)
        g = torch.Generator().manual_seed(3)
        inp["preconv_envmap"] = [2.0 * torch.rand(batch, 3, 16 >> i, 32 >> i, generator=g) for i in range(4)]
        inp["envbg"] = torch.rand(batch, 3, 64, 128, generator=g)
        inp["lightrot"] = torch.stack([rotation([0.0, 1.0, 0.0], 0.7 * (b + 1)) for b in range(batch)]).float()
        return inp
    inp = inputs(batch=batch)
    if mode == "train":
        inp["background"] = torch.rand(batch, 3, H, W, generator=torch.Generator().manual_seed(9))
        inp["is_fully_lit_frame"] = torch.tensor([True, False][:batch])
    return inp


def mode_config(mode):
    """config() for one fixture mode: noise_std = 0 in training, cal off for the environment map"""
    cfg = config()
    cfg["encoder"] = {**cfg["encoder"], "noise_std": 0.0}
    if mode == "envmap":
        cfg["cal"] = None
    return cfg


def functional_weights(preds, seed=101):
    """seeded fp64 weights of the pre-render functional sum_k <w_k, preds[k]> over PRIM_KEYS"""
    g = torch.Generator().manual_seed(seed)
    return {k: torch.randn(tuple(preds[k].shape), generator=g, dtype=torch.float64) for k in PRIM_KEYS}


def rgb_cotangent(shape, seed=77):
    return torch.randn(tuple(shape), generator=torch.Generator().manual_seed(seed), dtype=torch.float64)


def grad_param_names(model):
    """the first and last parameter (sorted by name) of the encoder, geometry decoder and Gaussian decoder"""
    names = sorted(n for n, _ in model.named_parameters())
    out = []
    for m in SUBMODULES:
        sub = [n for n in names if n.startswith(m + ".")]
        out += [sub[0], sub[-1]]
    return out


def summarise(t):
    """mean, std, max |.|, count and 256 evenly spaced samples of a tensor, fp64"""
    f = t.detach().double().reshape(-1).cpu()
    idx = torch.linspace(0, f.numel() - 1, 256, dtype=torch.float64).long()
    return np.concatenate([[f.mean().item(), f.std().item() if f.numel() > 1 else 0.0, f.abs().max().item(),
                            float(f.numel())], f[idx].numpy()])


def nrel_summary(a, b):
    """norm-wise relative difference of two summaries (statistics and samples, not the count)"""
    a, b = np.delete(np.asarray(a), 3), np.delete(np.asarray(b), 3)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300))
