"""Generate tests/golden/encoder_ref.npz by RUNNING the reference's own code on CPU (fp64):

  (a) a chain of two la.Conv2dWNUB(.., 4, 2, 1) layers (ca_code/nn/layers.py:276-327,472) with a LeakyReLU(0.2)
      between them, at small partial-tile sizes: parameters, input, output and every gradient;
  (b) the state_dict key / shape tables of the reference's Encoder(256, V) and GeomDecoder for a small V;
  (c) the reference Encoder's eval-mode embs_mu / embs_logvar at full size (1024^2 texture, B = 2) from the parameters
      and inputs of `encoder_recipe` below (only the outputs are stored: the recipe regenerates the rest);
  (d) a small-V GeomDecoder: its parameters and its output.

Encoder and GeomDecoder are executed from /root/reference/ca_code/models/rgca.py by slicing the classes out of the
file's AST at run time (the module itself cannot be imported here) — nothing is copied into this repository.
`encoder_recipe` imports nothing from the reference, so the tests use it directly.

Needs /root/reference; the .npz is committed.   Usage: python tests/golden/make_encoder_golden.py
"""
import ast
import json
import os
import sys
import warnings

import numpy as np
import torch as th

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "encoder_ref.npz")
SRC = "/root/reference/ca_code/models/rgca.py"

# fixture (c): Encoder(N_EMBS, N_VERTS) on a B x 3 x 1024 x 1024 texture
N_EMBS, N_VERTS, B_FULL = 256, 64, 2


def encoder_recipe(layout, n_verts=N_VERTS, batch=B_FULL, seed=20261015):
    """Seeded CPU parameters for an Encoder state_dict layout [(key, shape), ...] and its inputs (geom, color), fp32.
    Direction tensors ~ N(0, 1/fan_in), g = ||v|| * U(0.8, 1.2) (effective weights of unit-variance-preserving scale),
    biases ~ N(0, 0.05^2); geom ~ N(0, 1), color ~ U(0, 255).  Keys are drawn in sorted order, the g's last, so the
    result does not depend on the order in which a module registers its parameters."""
    gen = th.Generator().manual_seed(seed)
    sd = {}
    items = sorted((k, tuple(s)) for k, s in layout)
    for key, shape in [it for it in items if not it[0].endswith("weight_g")] + [it for it in items if it[0].endswith("weight_g")]:
        if key.endswith("weight_v"):
            fan_in = int(np.prod(shape[1:]))
            sd[key] = th.randn(shape, generator=gen) / np.sqrt(fan_in)
        elif key.endswith("weight_g"):
            v = sd[key[:-1] + "v"]
            sd[key] = v.norm() * (0.8 + 0.4 * th.rand(shape, generator=gen))
        else:
            sd[key] = 0.05 * th.randn(shape, generator=gen)
    geom = th.randn(batch, n_verts, 3, generator=gen)
    color = 255.0 * th.rand(batch, 3, 1024, 1024, generator=gen)
    return sd, geom, color


def _slice_class(tree, src, name):
    for node in tree.body:
        if isinstance(node, ast.ClassDef) and node.name == name:
            return ast.get_source_segment(src, node)
    raise KeyError(name)


def _jitter(mod):
    for m in mod.modules():
        if hasattr(m, "weight_g"):
            m.weight_g.data.mul_(1.0 + 0.3 * th.randn_like(m.weight_g))
        b = getattr(m, "bias", None)
        if b is not None:
            b.data.normal_(0, 0.3)


def main():
    if not os.path.isfile(SRC):
        sys.exit("needs /root/reference (build container only)")
    sys.path.insert(0, "/root/reference")
    warnings.filterwarnings("ignore")
    from typing import Dict

    import ca_code.nn.layers as la

    src = open(SRC).read()
    tree = ast.parse(src)
    ns = {"th": th, "nn": th.nn, "la": la, "Dict": Dict}
    for name in ("Encoder", "GeomDecoder"):
        exec(_slice_class(tree, src, name), ns)

    th.manual_seed(5521)
    d = {}

    # (a) la.Conv2dWNUB(4, 2, 1) chain 5 -> 11 (LeakyReLU) -> 7: 20x36 -> 10x18 -> 5x9 (partial tiles)
    net = th.nn.Sequential(la.Conv2dWNUB(5, 11, 10, 18, 4, 2, 1), th.nn.LeakyReLU(0.2),
                           la.Conv2dWNUB(11, 7, 5, 9, 4, 2, 1)).double()
    for m in net:
        la.glorot(m, 0.2)
    _jitter(net)
    x = th.randn(2, 5, 20, 36, dtype=th.float64, requires_grad=True)
    y = net(x)
    w = th.randn_like(y)
    params = [net[0].weight_v, net[0].weight_g, net[0].bias, net[2].weight_v, net[2].weight_g, net[2].bias]
    g = th.autograd.grad((y * w).sum(), [x] + params)
    d.update(cv_x=x, cv_y=y, cv_w=w, cv_gx=g[0])
    for i, (p, gp) in enumerate(zip(params, g[1:])):
        d["cv_p%d" % i], d["cv_gp%d" % i] = p, gp
    wv, wg = net[0].weight_v, net[0].weight_g
    assert wg.shape == (11, 1, 1, 1) and th.allclose(net[0].weight, wg * wv / wv.norm(), atol=1e-12)

    # (b) state_dict layouts
    V = 10
    layout = {"Encoder": [[k, list(v.shape)] for k, v in ns["Encoder"](256, V).state_dict().items()],
              "GeomDecoder": [[k, list(v.shape)] for k, v in ns["GeomDecoder"](256, th.randn(V, 3), 1.0).state_dict().items()]}
    d["layouts"] = np.array(json.dumps(layout))

    # (c) full-size Encoder, eval mode, recipe parameters, fp64
    enc = ns["Encoder"](N_EMBS, N_VERTS)
    sd, geom, color = encoder_recipe([(k, tuple(v.shape)) for k, v in enc.state_dict().items()])
    enc.load_state_dict(sd)
    enc = enc.double().eval()
    with th.no_grad():
        out = enc(geom.double(), color.double())
    d.update(enc_mu=out["embs_mu"], enc_logvar=out["embs_logvar"])
    assert th.equal(out["embs"], out["embs_mu"])

    # (d) GeomDecoder, n_embs 16, 12 vertices
    gd = ns["GeomDecoder"](16, 10.0 * th.randn(12, 3), 2.5).double()
    _jitter(gd)
    embs = th.randn(3, 16, dtype=th.float64)
    with th.no_grad():
        d["gd_geom"] = gd(embs)["face_geom"]
    d["gd_embs"] = embs
    for k, v in gd.state_dict().items():
        d["gd_p_" + k] = v
    d["gd_names"] = np.array(json.dumps(list(gd.state_dict().keys())))

    outd = {k: (v.detach().numpy() if isinstance(v, th.Tensor) else v) for k, v in d.items()}
    np.savez_compressed(OUT, **outd)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
