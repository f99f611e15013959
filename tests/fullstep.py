"""CPU oracle of the WHOLE benchmarked step (bench.py's `gpu_step`): SG shade + colour compose -> EWA projection ->
bin/sort -> one 4-channel blend (rgb + depth) -> rgca.AutoEncoder.render post-processing, forward and backward with
v_out = 1 (SURVEY.md section 8d), from the C oracle's pieces (oracle/*.c).  Test infrastructure only.

Reference call sequence restated: ca_code/models/rgca.py:557-575 (shade + compose), ca_code/utils/render_gsplat.py:41-106
(project, rasterise rgb, rasterise depth-as-colour), rgca.py:112-151 (alpha from the DETACHED final_T, depth divided by
alpha.clamp(0.05, 1))."""
import numpy as np


def oracle_step(orc, u, cam, li, H, W, bw=16):
    """u: dict of numpy arrays with bench.FIELDS names; cam: dict(Rt [3,4], intr (fx,fy,cx,cy)); li: numpy lights.
    Returns dict(rgb [3,H,W], alpha [H,W], depth [H,W], n_isect, grads {field: array})."""
    f32 = np.float32
    fx, fy, cx, cy = cam["intr"]
    V = np.asarray(cam["Rt"], f32)
    raw = u["lobe_dirs"].astype(np.float64)
    nrm_len = np.linalg.norm(raw, axis=-1, keepdims=True)
    nrm = (raw / nrm_len).astype(f32)
    spec = orc.sg_fwd(nrm[None], u["sigma"][None], li["light_intensity"], li["light_pos"], u["primpos"][None],
                      li["n_lights"], 0)[0]
    vis = u["spec_vis"].reshape(-1, 1)
    pre = np.maximum(u["diff_color"], 0) + spec * vis
    color = np.maximum(pre, 0).astype(f32)
    p = orc.project_fwd(u["primpos"], u["primscale"], 1.0, u["primqvec"], V, fx, fy, cx, cy, H, W, bw, 0.1)
    b = orc.bin_and_sort(p["xys"], p["depths"], p["radii"], p["num_tiles_hit"], H, W, bw)
    opac = (u["opacity"].reshape(-1) * p["compensation"]).astype(f32)
    col4 = np.concatenate([color, p["depths"][:, None]], 1).astype(f32)
    z4 = np.zeros(4, f32)
    out4, Ts, fi = orc.rasterize_fwd(H, W, bw, b["gaussian_ids_sorted"], b["tile_bins"], p["xys"], p["conics"], col4,
                                     opac, z4)
    alpha = (1.0 - Ts).astype(f32)
    inv_a = (1.0 / np.clip(alpha, 0.05, 1.0)).astype(f32)
    rgb = np.transpose(out4[..., :3], (2, 0, 1))
    depth = out4[..., 3] * inv_a
    # backward, loss = sum(rgb) + sum(depth); alpha is detached (rgca.py:137)
    v_out4 = np.ones((H, W, 4), f32)
    v_out4[..., 3] = inv_a
    g = orc.rasterize_bwd(H, W, bw, b["gaussian_ids_sorted"], b["tile_bins"], p["xys"], p["conics"], col4, opac, z4,
                          Ts, fi, v_out4, np.zeros((H, W), f32))
    v_xy, v_conic, v_col4, v_opeff = g
    v_opeff = v_opeff.reshape(-1)
    pb = orc.project_bwd(u["primpos"], u["primscale"], 1.0, u["primqvec"], V, fx, fy, p["cov3d"], p["radii"], p["conics"],
                         p["compensation"], v_xy, v_col4[:, 3].copy(), v_conic, v_opeff * u["opacity"].reshape(-1))
    g_color = v_col4[:, :3] * (pre >= 0)
    g_diff = g_color * (u["diff_color"] >= 0)
    g_spec = g_color * vis
    g_vis = (g_color * spec).sum(-1)
    gd, gs, _ = orc.sg_bwd(nrm[None], u["sigma"][None], li["light_intensity"], li["light_pos"], u["primpos"][None],
                           li["n_lights"], g_spec[None].astype(f32), 0, want_light_grad=False)
    gd = gd[0].astype(np.float64)
    n64 = nrm.astype(np.float64)
    g_raw = (gd - n64 * (n64 * gd).sum(-1, keepdims=True)) / nrm_len
    grads = dict(primpos=pb["v_mean3d"], primqvec=pb["v_quat"], primscale=pb["v_scale"],
                 opacity=(v_opeff * p["compensation"]).reshape(u["opacity"].shape), diff_color=g_diff.astype(f32),
                 lobe_dirs=g_raw.astype(f32), sigma=gs[0], spec_vis=g_vis.reshape(u["spec_vis"].shape).astype(f32))
    return dict(rgb=rgb, alpha=alpha, depth=depth, n_isect=int(b["num_intersects"]), grads=grads,
                bins=b["tile_bins"], gids=b["gaussian_ids_sorted"])


def oracle_shared_view(orc, means, scales, quats, opacity, colors, bg, viewmat, intr, H, W, v_rgb, v_depth=None,
                       v_alpha=None, bw=16):
    """One view, C colour sets against one projection and one binning (gsplat/olat.py render_shared), restated per
    condition with the C oracle, whose blend takes at most 8 channels: condition 0 is blended with the depth channel
    (4 channels, background [bg, bg[0]] as render_fused), conditions 1.. with 3; the backward runs on the oracle's own
    forward state, only condition 0 carries the alpha gradient, and the geometry gradients are summed over the
    conditions before ONE projection backward.  colors [C,G,3]; v_rgb [C,H,W,3]; v_depth / v_alpha [H,W] or None.
    Returns dict(rgb [C,H,W,3], depth_raw [H,W], alpha [H,W], n_isect, grads {means3d, scales, quats, opacity [G,1],
    colors [C,G,3]})."""
    f32 = np.float32
    fx, fy, cx, cy = intr
    viewmat = np.asarray(viewmat, f32)
    C, G = colors.shape[:2]
    p = orc.project_fwd(means, scales, 1.0, quats, viewmat, fx, fy, cx, cy, H, W, bw, 0.1)
    b = orc.bin_and_sort(p["xys"], p["depths"], p["radii"], p["num_tiles_hit"], H, W, bw)
    gids, bins = b["gaussian_ids_sorted"], b["tile_bins"]
    opac = (opacity.reshape(-1) * p["compensation"]).astype(f32)
    bg = np.asarray(bg, f32)
    zero_a = np.zeros((H, W), f32)
    col4 = np.concatenate([colors[0], p["depths"][:, None]], 1).astype(f32)
    bg4 = np.append(bg, bg[0]).astype(f32)
    out4, Ts, fi = orc.rasterize_fwd(H, W, bw, gids, bins, p["xys"], p["conics"], col4, opac, bg4)
    alpha = (1.0 - Ts).astype(f32)
    if callable(v_depth):  # a weight that depends on the (detached) alpha
        v_depth = v_depth(alpha)
    v4 = np.concatenate([v_rgb[0], (zero_a if v_depth is None else v_depth)[..., None]], -1).astype(f32)
    v_xy, v_conic, v_col4, v_opeff = orc.rasterize_bwd(H, W, bw, gids, bins, p["xys"], p["conics"], col4, opac, bg4, Ts,
                                                       fi, v4, zero_a if v_alpha is None else v_alpha)
    rgb, v_colors = [out4[..., :3]], [v_col4[:, :3]]
    for c in range(1, C):
        img, _, _ = orc.rasterize_fwd(H, W, bw, gids, bins, p["xys"], p["conics"], colors[c], opac, bg)
        g = orc.rasterize_bwd(H, W, bw, gids, bins, p["xys"], p["conics"], colors[c], opac, bg, Ts, fi, v_rgb[c], zero_a)
        rgb.append(img)
        v_colors.append(g[2])
        v_xy, v_conic, v_opeff = v_xy + g[0], v_conic + g[1], v_opeff + g[3]
    v_opeff = v_opeff.reshape(-1)
    pb = orc.project_bwd(means, scales, 1.0, quats, viewmat, fx, fy, p["cov3d"], p["radii"], p["conics"],
                         p["compensation"], v_xy, v_col4[:, 3].copy(), v_conic, v_opeff * opacity.reshape(-1))
    grads = dict(means3d=pb["v_mean3d"], scales=pb["v_scale"], quats=pb["v_quat"],
                 opacity=(v_opeff * p["compensation"]).reshape(G, 1), colors=np.stack(v_colors))
    return dict(rgb=np.stack(rgb), depth_raw=out4[..., 3], alpha=alpha, n_isect=int(b["num_intersects"]), grads=grads)


def oracle_olat_step(orc, u, cams, li, H, W, bw=16):
    """CPU oracle of bench.py's OLAT step (`OlatWorkload.compute`): oracle_step per lighting condition c, i.e. the
    L = 1 SG shade of light c + colour compose, blended against the view's one projection and binning
    (oracle_shared_view); condition 0 also carries the depth, divided by the DETACHED alpha.clamp(0.05, 1).  Loss =
    sum of every rgb image and every depth image (v_out = 1).  u: bench.FIELDS arrays; cams: list of dict(Rt, intr);
    li: numpy lights with one light per condition.  Returns dict(rgb [V,C,H,W,3], alpha [V,H,W], depth [V,H,W],
    n_isect [V], grads {field: sum over conditions and views})."""
    f32 = np.float32
    C = li["light_intensity"].shape[1]
    G = u["primpos"].shape[0]
    raw = u["lobe_dirs"].astype(np.float64)
    nrm_len = np.linalg.norm(raw, axis=-1, keepdims=True)
    nrm = (raw / nrm_len).astype(f32)
    vis = u["spec_vis"].reshape(-1, 1)
    one = np.ones(1, np.int32)
    lights = [(li["light_intensity"][:, c:c + 1], li["light_pos"][:, c:c + 1]) for c in range(C)]
    specs = [orc.sg_fwd(nrm[None], u["sigma"][None], lv, lp, u["primpos"][None], one, 0)[0] for lv, lp in lights]
    pres = [np.maximum(u["diff_color"], 0) + sp * vis for sp in specs]
    colors = np.stack([np.maximum(pre, 0) for pre in pres]).astype(f32)  # [C,G,3]
    rgbs, alphas, depths, n_isect = [], [], [], []
    g_col = np.zeros((C, G, 3), f32)
    geo = {k: np.zeros_like(u[k]) for k in ("primpos", "primqvec", "primscale", "opacity")}
    inv_a = lambda alpha: (1.0 / np.clip(alpha, 0.05, 1.0)).astype(f32)
    for cam in cams:
        r = oracle_shared_view(orc, u["primpos"], u["primscale"], u["primqvec"], u["opacity"], colors, np.zeros(3, f32),
                               cam["Rt"], cam["intr"], H, W, np.ones((C, H, W, 3), f32), v_depth=inv_a, bw=bw)
        rgbs.append(r["rgb"])
        alphas.append(r["alpha"])
        depths.append(r["depth_raw"] * inv_a(r["alpha"]))
        n_isect.append(r["n_isect"])
        g_col += r["grads"]["colors"]
        for k, n in (("primpos", "means3d"), ("primqvec", "quats"), ("primscale", "scales"), ("opacity", "opacity")):
            geo[k] += r["grads"][n].reshape(geo[k].shape)
    g_diff = np.zeros_like(u["diff_color"])
    g_vis = np.zeros(G, f32)
    gd_sum = np.zeros((G, 3), np.float64)
    g_sigma = np.zeros_like(u["sigma"])
    for c, (lv, lp) in enumerate(lights):
        g_color = g_col[c] * (pres[c] >= 0)
        g_diff += g_color * (u["diff_color"] >= 0)
        g_vis += (g_color * specs[c]).sum(-1)
        gd, gs, _ = orc.sg_bwd(nrm[None], u["sigma"][None], lv, lp, u["primpos"][None], one,
                               (g_color * vis)[None].astype(f32), 0, want_light_grad=False)
        gd_sum += gd[0]
        g_sigma += gs[0]
    n64 = nrm.astype(np.float64)
    g_raw = (gd_sum - n64 * (n64 * gd_sum).sum(-1, keepdims=True)) / nrm_len
    grads = dict(geo, diff_color=g_diff.astype(f32), lobe_dirs=g_raw.astype(f32), sigma=g_sigma,
                 spec_vis=g_vis.reshape(u["spec_vis"].shape).astype(f32))
    return dict(rgb=np.stack(rgbs), alpha=np.stack(alphas), depth=np.stack(depths), n_isect=n_isect, grads=grads)
