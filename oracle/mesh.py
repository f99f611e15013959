"""CPU oracle of the body render (mesh_oracle.c) — TEST INFRASTRUCTURE ONLY.

numpy-in / numpy-out wrappers over ``libmesh_oracle.so``, which gcc builds from ``mesh_oracle.c`` with
``-ffp-contract=off``, the same flags as ``liboracle.so``. That flag keeps the fp32 rasteriser bit-exact with
csrc/mesh_raster.cu.

Parity: PARITY UNPINNED. drtk is a third-party dependency outside the reference tree. The rasteriser, sampling
and edge-gradient conventions are the project's (DESIGN.md R9''). The reference's own RenderLayer code is pinned by
tests/golden/mesh_render_ref.npz.
"""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


def build(force: bool = False) -> str:
    so = os.path.join(_HERE, "libmesh_oracle.so")
    src = os.path.join(_HERE, "mesh_oracle.c")
    if force or not os.path.exists(so) or os.path.getmtime(src) > os.path.getmtime(so):
        subprocess.check_call(["gcc", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-Wall", "-o", so, src, "-lm"])
    return so


def lib():
    global _LIB
    if _LIB is None:
        _LIB = ctypes.CDLL(build())
    return _LIB


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p) if a is not None else None


def _f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def _i32(a):
    return np.ascontiguousarray(a, dtype=np.int32)


def mesh_raster(v_pix, vi, H, W):
    """index image [B,H,W] int32 of v_pix [B,V,3], vi [F,3]: the kernel's fp32 arithmetic, bit-exact"""
    v_pix, vi = _f32(v_pix), _i32(vi)
    B, V = v_pix.shape[:2]
    out = np.zeros((B, H, W), np.int32)
    c = ctypes
    lib().orc_mesh_raster(c.c_int(B), c.c_int(V), c.c_int(vi.shape[0]), c.c_int(H), c.c_int(W), _p(v_pix), _p(vi),
                          _p(out))
    return out


def _mesh_args(v_pix, vi, vti, vt, tex, index_img):
    v_pix, vi, vti, vt, tex, index_img = _f32(v_pix), _i32(vi), _i32(vti), _f32(vt), _f32(tex), _i32(index_img)
    B, V = v_pix.shape[:2]
    C, Ht, Wt = tex.shape[1:]
    H, W = index_img.shape[1:]
    c = ctypes
    dims = [c.c_int(B), c.c_int(V), c.c_int(vi.shape[0]), c.c_int(H), c.c_int(W), c.c_int(C), c.c_int(Ht), c.c_int(Wt)]
    return (B, V, C, H, W, Ht, Wt), dims, [_p(v_pix), _p(vi), _p(vti), _p(vt), _p(tex), _p(index_img)], (
        v_pix, vi, vti, vt, tex, index_img)


def mesh_render_fwd(v_pix, vi, vti, vt, tex, index_img):
    """fp64 {depth_img, bary_img, vt_img, mask, render} at the index image (vt as RenderLayer holds it)"""
    (B, V, C, H, W, Ht, Wt), dims, ptrs, keep = _mesh_args(v_pix, vi, vti, vt, tex, index_img)
    out = dict(depth_img=np.zeros((B, H, W)), bary_img=np.zeros((B, 3, H, W)), vt_img=np.zeros((B, 2, H, W)),
               mask=np.zeros((B, 1, H, W)), render=np.zeros((B, C, H, W)))
    lib().orc_mesh_render_fwd(*dims, *ptrs, *[_p(out[k]) for k in ("depth_img", "bary_img", "vt_img", "mask",
                                                                    "render")])
    return out


def mesh_render_bwd(v_pix, vi, vti, vt, tex, index_img, g_render, edge_grad=True):
    """fp64 (g_v_pix [B,V,3], g_tex [B,C,Ht,Wt]) of sum(g_render * render) at the index image"""
    (B, V, C, H, W, Ht, Wt), dims, ptrs, keep = _mesh_args(v_pix, vi, vti, vt, tex, index_img)
    g_render = _f32(g_render)
    g_v, g_t = np.zeros((B, V, 3)), np.zeros((B, C, Ht, Wt))
    lib().orc_mesh_render_bwd(*dims, *ptrs, _p(g_render), ctypes.c_int(int(edge_grad)), _p(g_v), _p(g_t))
    return g_v, g_t
