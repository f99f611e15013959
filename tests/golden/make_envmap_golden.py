"""Generate tests/golden/envmap_compose_ref.npz from the REFERENCE's own `rotate_envmap_mat` and `compose_envmap`
(ca_code/utils/envmap.py:141-166, 325-345), run on the CPU in fp32 (the reference builds its blur kernel in fp32, so
fp64 inputs raise).  Nothing is copied: the functions are imported from a reference checkout.

The inputs are not stored: `case_inputs` rebuilds them from numpy seeds (PCG64 streams are stable across numpy
versions), and tests/test_envmap_compose_gpu.py reads the fixture through `golden_case` from this file.  Stored: the
composite of each case outside the mirror ball, each distinct mirror ball and rotated probe once (see PAIRS), and the
mirror-ball mask; quantised and LZMA-compressed by `encode` (the fixture is 0.7 MB).

Cases (B = 2 each; probes P are 64x128, Q are 32x64, values 0.6 .. 1.4):
  a216x240   identity camera, centred, alpha 0 | central ray next to the +y pole (v = 1; every u around it, so the
             u = +-1 seam too), off-centre principal point with fx != fy, alpha 1
  b200x200   the image is exactly the mirror ball: central ray next to the -y pole (v = -1) | a random rotation scaled
             by 1.3, so the unnormalised mirror-ball directions leave [-1, 1] and acos gives NaN (the reference clamps
             nothing); smooth alpha with exact 0 and 1 regions
  c203x331   a ragged image with the probes and rotations of a216x240 (so the same mirror balls) and other
             intrinsics (off-centre, fx != fy) and alpha

Usage: python tests/golden/make_envmap_golden.py /path/to/goliath-checkout
"""
import lzma
import os
import sys

import numpy as np

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "envmap_compose_ref.npz")
CASES = ("a216x240", "b200x200", "c203x331")
QSCALE = float(2 ** 16)   # composite and rotated probes
BALL_QSCALE = float(2 ** 15)  # mirror balls: probe values >= 0.6, so the bar there is >= 8e-5


def _rot(axis, deg):
    t = np.deg2rad(deg)
    c, s = np.cos(t), np.sin(t)
    if axis == "x":
        return np.array([[1, 0, 0], [0, c, -s], [0, s, c]])
    if axis == "y":
        return np.array([[c, 0, s], [0, 1, 0], [-s, 0, c]])
    return np.array([[c, -s, 0], [s, c, 0], [0, 0, 1]])


def _random_rot(rng):
    q = rng.standard_normal(4)
    w, x, y, z = q / np.linalg.norm(q)
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


def _camera(R, fx, fy, cx, cy, t=(0.0, 0.0, 1000.0)):
    K = np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1]], np.float32)
    Rt = np.concatenate([np.asarray(R, np.float64), np.asarray(t, np.float64)[:, None]], 1).astype(np.float32)
    return K, Rt


def _smooth(rng, shape, lo, hi, cycles=(0.3, 1.5)):
    """a smooth random image (a few random waves per channel of `cycles` periods per image), the kind of content a
    render or a light probe has"""
    B, C, H, W = shape
    y, x = np.mgrid[0:H, 0:W].astype(np.float64)
    out = np.zeros(shape)
    for b in range(B):
        for c in range(C):
            for _ in range(4):
                fy, fx = rng.uniform(*cycles, 2) * 2 * np.pi / np.array([H, W])
                out[b, c] += rng.uniform(0.2, 1.0) * np.sin(fy * y + fx * x + rng.uniform(0, 2 * np.pi))
    out = (out - out.min()) / (out.max() - out.min())
    return (lo + (hi - lo) * out).astype(np.float32)


def _probe(seed, He, We):
    """one light probe [3,He,We]: smooth, with values above 1 (clamped in the image, not in the mirror ball)"""
    return _smooth(np.random.default_rng(seed), (1, 3, He, We), 0.6, 1.4)[0]


# (probe, rotation) of each batch item.  The mirror ball depends on nothing else, so items that share a pair share their
# 200x200 ball (and their rotated probe); the fixture stores each distinct ball once.
PAIRS = (("P1", "I"), ("P2", "Rx90"), ("Q1", "Rx-90"), ("Q2", "scaled"))
CASE_PAIRS = {"a216x240": (0, 1), "b200x200": (2, 3), "c203x331": (0, 1)}


def _rotation(name):
    return {"I": np.eye(3), "Rx90": _rot("x", 90), "Rx-90": _rot("x", -90),
            "scaled": 1.3 * _random_rot(np.random.default_rng(1345))}[name]


def case_inputs(name):
    """render [2,3,H,W], alpha [2,1,H,W], envbg [2,3,He,We], K [2,3,3], Rt [2,3,4] of one case, from fixed seeds"""
    rng = np.random.default_rng(325 + CASES.index(name))
    H, W = {"a216x240": (216, 240), "b200x200": (200, 200), "c203x331": (203, 331)}[name]
    render = _smooth(rng, (2, 3, H, W), 0.0, 1.0, (0.2, 0.8))
    a = np.clip(_smooth(rng, (2, 1, H, W), -0.3, 1.3, (0.2, 0.8)), 0.0, 1.0)  # with exact 0 and 1 regions
    pairs = [PAIRS[i] for i in CASE_PAIRS[name]]
    probes = {"P1": (1, 64, 128), "P2": (2, 64, 128), "Q1": (3, 32, 64), "Q2": (4, 32, 64)}
    envbg = np.stack([_probe(*probes[p]) for p, _ in pairs])
    R = [_rotation(r) for _, r in pairs]
    if name == "a216x240":
        a[0], a[1] = 0.0, 1.0
        intr = [(300.0, 300.0, 0.5 * W, 0.5 * H), (260.0, 410.0, 30.3, 190.7)]
    elif name == "b200x200":
        intr = [(280.0, 320.0, 100.61, 99.58), (300.0, 300.0, 99.37, 100.21)]
    else:
        intr = [(350.0, 270.0, 265.2, 31.4), (330.0, 300.0, 150.3, 110.9)]
    cams = [_camera(r, *k) for r, k in zip(R, intr)]
    K = np.stack([c[0] for c in cams])
    Rt = np.stack([c[1] for c in cams])
    return dict(render=render, alpha=a, envbg=envbg, K=K, Rt=Rt)


def encode(d, key, x, scale=QSCALE):
    """store fp32 image x under `key`: the second differences along the rows of round(x * scale) as int32, split into
    their four byte planes and LZMA-compressed (d[key], with the shape in d[key + "_shape"]), and the packed NaN mask
    (d[key + "_nan"], compressed too).  A step of 2^-16 keeps every value within 7.6e-6 of the reference's (2^-15 and 1.5e-5 for the
    mirror balls, whose values are >= 0.6); on smooth images the differences are small, so the planes compress well."""
    nan = np.isnan(x)
    q = np.round(np.where(nan, 0.0, x).astype(np.float64) * scale).astype(np.int64)
    dd = np.diff(np.diff(q, axis=-1, prepend=0), axis=-1, prepend=0).astype("<i4")
    planes = np.moveaxis(dd[..., None].view(np.uint8), -1, 0).tobytes()
    d[key] = np.frombuffer(lzma.compress(planes, preset=9 | lzma.PRESET_EXTREME), np.uint8)
    d[key + "_shape"] = np.array(x.shape, np.int64)
    d[key + "_nan"] = np.frombuffer(lzma.compress(np.packbits(nan.reshape(-1)).tobytes()), np.uint8)


def decode(z, key, scale=QSCALE):
    shape = tuple(int(v) for v in z[key + "_shape"])
    planes = np.frombuffer(lzma.decompress(z[key].tobytes()), np.uint8).reshape((4,) + shape)
    dd = np.ascontiguousarray(np.moveaxis(planes, 0, -1)).view("<i4")[..., 0]
    q = np.cumsum(np.cumsum(dd.astype(np.int64), axis=-1), axis=-1)
    x = (q / scale).astype(np.float32)
    nan = np.frombuffer(lzma.decompress(z[key + "_nan"].tobytes()), np.uint8)
    x[np.unpackbits(nan, count=x.size).reshape(shape).astype(bool)] = np.nan
    return x


def ball_region(H, W, mask):
    """[H,W] bool: the pixels of the mirror ball (zsq < 1) in the bottom-right 200x200 corner"""
    m = np.zeros((H, W), bool)
    m[-200:, -200:] = mask.astype(bool)
    return m


def golden_case(z, name):
    """the reference's outputs of one case, decoded: out [2,3,H,W] and rot [2,3,He,We]"""
    out = decode(z, name + "_out")
    inside = ball_region(out.shape[2], out.shape[3], z["mask"])
    rot = []
    for b, k in enumerate(CASE_PAIRS[name]):
        ball = decode(z, "ball%d" % k, BALL_QSCALE)
        out[b][:, inside] = ball[:, inside[-200:, -200:]]
        rot.append(decode(z, "rot%d" % k))
    return out, np.stack(rot)


def main():
    if len(sys.argv) != 2 or not os.path.isdir(os.path.join(sys.argv[1], "ca_code")):
        sys.exit(__doc__)
    sys.path.insert(0, sys.argv[1])
    import torch as th
    from ca_code.utils.envmap import compose_envmap, rotate_envmap_mat

    d = {}
    balls = {}
    for name in CASES:
        x = case_inputs(name)
        t = {k: th.from_numpy(v) for k, v in x.items()}
        out = compose_envmap(t["render"], t["alpha"], t["envbg"], t["K"], t["Rt"]).numpy()
        # the mirror mask, read back through the composite: render 1, alpha 1, a black environment -> out = 1 - mask
        m = (compose_envmap(th.ones_like(t["render"]), th.ones_like(t["alpha"]), th.zeros_like(t["envbg"]), t["K"],
                            th.eye(3).expand(2, 3, 3)) == 0).numpy()[0, 0, -200:, -200:]
        assert "mask" not in d or np.array_equal(d["mask"], m)
        d["mask"] = m.astype(np.uint8)
        inside = ball_region(out.shape[2], out.shape[3], m)
        for b, k in enumerate(CASE_PAIRS[name]):
            ball = out[b, :, -200:, -200:]
            if k in balls:  # the same probe and rotation: the ball must be the stored one, bit for bit
                assert np.array_equal(balls[k][:, m], ball[:, m], equal_nan=True), (name, b)
            else:
                balls[k] = ball.copy()
                encode(d, "ball%d" % k, np.where(m, ball, 0.0).astype(np.float32), BALL_QSCALE)
                rot = rotate_envmap_mat(t["envbg"][b], t["Rt"][b, :3, :3]).numpy()
                encode(d, "rot%d" % k, rot)
        rest = out.copy()
        rest[:, :, inside] = 0.0  # stored once per (probe, rotation) in ball<k>
        encode(d, "%s_out" % name, rest)
        print("%s: out %s, NaN %d, mask %d px" % (name, tuple(out.shape), int(np.isnan(out).sum()), int(m.sum())))
    np.savez(OUT, **d)  # the arrays are LZMA streams already
    print("wrote %s (%d bytes)" % (OUT, os.path.getsize(OUT)))


if __name__ == "__main__":
    main()
