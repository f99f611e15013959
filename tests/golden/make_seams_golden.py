"""Generate tests/golden/seams_ref.npz with the REFERENCE's own ca_code/utils/seams.py (`SeamSampler`: impaint_batch,
resample_tex) and ca_code/utils/geom.py (`sample_uv`), imported from /root/reference (build container only), on CPU
in fp64, on small synthetic seam data:
  - a dst texel that is also the src of another pair, and one src read by several dst (no duplicate dst: the
    reference's index_put leaves those undefined);
  - uvs outside [0, 1] (border padding) and seam weights of 0, 1 and in between;
  - vt on and beyond the map edge, v2uv rows padded by repeating their first entry (compute_v2uv).
Stores inputs, outputs and autograd gradients.

Usage: python tests/golden/make_seams_golden.py"""
import os
import sys
import types
from unittest.mock import MagicMock

import numpy as np
import torch as th

sys.path.insert(0, "/root/reference")
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "seams_ref.npz")


def main():
    for name in ("pytorch3d", "pytorch3d.renderer", "pytorch3d.renderer.mesh", "pytorch3d.renderer.mesh.rasterize_meshes",
                 "pytorch3d.structures", "pytorch3d.io", "drtk", "addict", "omegaconf", "igl", "trimesh"):
        if name not in sys.modules:
            try:
                __import__(name)
            except Exception:
                sys.modules[name] = MagicMock() if name != "addict" else types.SimpleNamespace(Dict=dict)
    from ca_code.utils import geom, seams

    g = th.Generator().manual_seed(1441)
    B, C, H, W = 2, 3, 12, 10
    # seam pairs (row, col): (3,4) is a dst and also the src of (0,0); (7,7) is the src of three dst texels
    dst = th.tensor([[0, 0], [3, 4], [5, 1], [9, 9], [11, 0], [2, 8], [6, 6]])
    src = th.tensor([[3, 4], [7, 7], [7, 7], [7, 7], [0, 9], [10, 2], [1, 1]])
    uvs = (th.rand(H, W, 2, generator=g, dtype=th.float64) * 1.4 - 0.2)   # some outside [0, 1]
    uvs[0, 0] = th.tensor([0.0, 0.0]); uvs[0, 1] = th.tensor([1.0, 1.0]); uvs[0, 2] = th.tensor([-0.5, 1.5])
    weights = th.rand(H, W, generator=g, dtype=th.float64)
    weights[1, :4] = 0.0
    weights[2, :4] = 1.0
    sampler = seams.SeamSampler(dict(dst_ij=dst, src_ij=src, uvs=uvs, weights=weights))

    tex = th.randn(B, C, H, W, generator=g, dtype=th.float64).requires_grad_()
    imp = sampler.impaint(tex.clone())
    res = sampler.resample(tex)
    fwd = sampler.forward(tex.clone())
    chain = sampler.resample(sampler.resample(sampler.impaint(tex.clone())))   # mesh_vae.py:611-613
    ws = {k: th.randn(t.shape, generator=g, dtype=th.float64) for k, t in
          (("impaint", imp), ("resample", res), ("forward", fwd), ("chain", chain))}
    grads = {}
    for k, t in (("impaint", imp), ("resample", res), ("forward", fwd), ("chain", chain)):
        (grads[k],) = th.autograd.grad((t * ws[k]).sum(), [tex])

    # sample_uv: vt on / beyond the edges, v2uv with padded duplicates
    n_uv, V = 9, 5
    vt = th.rand(n_uv, 2, generator=g, dtype=th.float64)
    vt[0] = th.tensor([0.0, 0.0]); vt[1] = th.tensor([1.0, 1.0]); vt[2] = th.tensor([1.08, 0.5])
    vt[3] = th.tensor([-0.05, -0.1])
    v2uv = th.tensor([[0, 4, 0, 0], [1, 2, 3, 1], [5, 5, 5, 5], [6, 7, 8, 6], [2, 3, 2, 2]])
    uvmap = th.randn(B, C, H, W, generator=g, dtype=th.float64).requires_grad_()
    sv = geom.sample_uv(uvmap, vt, v2uv)
    wsv = th.randn(sv.shape, generator=g, dtype=th.float64)
    (g_uvmap,) = th.autograd.grad((sv * wsv).sum(), [uvmap])

    d = dict(dst_ij=dst, src_ij=src, uvs=uvs, weights=weights, tex=tex, impaint=imp, resample=res, forward=fwd,
             chain=chain, vt=vt, v2uv=v2uv, uvmap=uvmap, sample_uv=sv, w_sample_uv=wsv, g_uvmap=g_uvmap)
    d.update({"w_" + k: t for k, t in ws.items()})
    d.update({"g_" + k: t for k, t in grads.items()})
    np.savez_compressed(OUT, **{k: t.detach().numpy() for k, t in d.items()})
    print("wrote %s (%d bytes)" % (OUT, os.path.getsize(OUT)))


if __name__ == "__main__":
    main()
