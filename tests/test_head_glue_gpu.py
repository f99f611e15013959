"""The head view's render node (gsplat.fused._RenderBuckets with finish=True: the blend kernels finish the view, one
per-Gaussian backward pass) against the composition it replaces, rebuilt here from the kept entry points and torch
ops: gb_project_gaussians_fwd -> gb_bin_tiles_buckets -> gb_rasterize_ranked_fwd_sort_lists -> 1 - final_Ts ->
gb_render_finish_fwd, and back through gb_render_finish_bwd -> gb_rasterize_ranked_bwd_lists -> gb_splat_grad_unpack
-> gb_project_gaussians_bwd.

- rgb, alpha, depth, the sorted ids, final_Ts, final_idx, the hit counts and the written hit-list entries are identical
  bit for bit; the five input gradients agree up to the order of the blend backward's atomic adds;
- given the same accumulated blend gradients, gb_splat_project_bwd gives gb_splat_grad_unpack +
  gb_project_gaussians_bwd's gradients bit for bit;
- with g_rgb or g_depth absent, under CUDA-graph replay, at a Gaussian count that is not a multiple of 4, and at 2^20
  Gaussians (tiles longer than the forward's shared-memory sort)."""
import numpy as np
import pytest
import torch

from util import assert_close, t2n

pytestmark = pytest.mark.gpu

GRADS = ("means3d", "scales", "quats", "opacity", "colors")


def _scene(cuda, G, cam_k):
    import bench
    from goliath_b200 import synthetic

    # copies, not views of the packed buffer: with G not a multiple of 4 the fields there are not 16-byte aligned
    u = {k: v.clone() for k, v in bench.unpack(bench.packed_scene(G).to(cuda)).items()}
    c = synthetic.ring_camera(cam_k, img_h=bench.H, img_w=bench.W)
    g = torch.Generator(device="cpu").manual_seed(cam_k)
    return dict(means3d=u["primpos"], scales=u["primscale"], quats=u["primqvec"], opacity=u["opacity"],
                colors=u["diff_color"],
                viewmat=c["viewmat"].to(cuda), intr=(c["fx"], c["fy"], c["cx"], c["cy"]),
                background=torch.rand(3, generator=g).to(cuda), H=bench.H, W=bench.W, cap=max(8 * G, 1 << 20),
                g_rgb=torch.randn(3, bench.H, bench.W, generator=g).to(cuda),
                g_depth=torch.randn(1, bench.H, bench.W, generator=g).to(cuda))


def _parent(sc, use_rgb=True, use_depth=True, acc=None):
    """The replaced composition.  Returns the view, the blend's internals and the five input gradients."""
    from goliath_b200 import _lib
    from goliath_b200.gsplat import utils as gu
    from goliath_b200.gsplat.project import _project_fwd

    L = _lib.lib()
    dev = sc["means3d"].device
    st = _lib.stream_ptr(dev)
    p = _lib.ptr
    f32, i32 = dict(device=dev, dtype=torch.float32), dict(device=dev, dtype=torch.int32)
    G, H, W, cap = sc["means3d"].shape[0], sc["H"], sc["W"], sc["cap"]
    fx, fy, cx, cy = sc["intr"]
    xys, depths, radii, conics, comp, _, cov3d = _project_fwd(sc["means3d"], sc["scales"], sc["quats"], sc["viewmat"],
                                                              1.0, fx, fy, cx, cy, H, W, 16, 0.1)
    tb = gu._tile_bounds(H, W, 16)
    T = tb[0] * tb[1]
    bins, order = torch.empty(T, 2, **i32), torch.empty(T, **i32)
    ranks, bucket, records, gids = (torch.empty(cap, **i32), torch.empty(cap, **i32), torch.empty(G, 12, **f32),
                                    torch.empty(G, **i32))
    n, ovf = torch.zeros(1, **i32), torch.zeros(1, **i32)
    ws = torch.empty(L.gb_bin_tiles_workspace_bytes(G, T, cap), dtype=torch.uint8, device=dev)
    _lib.check(L.gb_bin_tiles_buckets(G, p(xys), p(depths), p(radii), p(conics), p(sc["colors"]), p(sc["opacity"]),
                                      p(comp), H, W, 16, cap, p(bins), p(order), p(ranks), p(bucket), p(records),
                                      p(gids), p(n), p(ovf), p(ws), None, st), "bin_tiles_buckets")
    bg4 = torch.cat([sc["background"], sc["background"][:1]])
    out4, final_Ts, final_idx = torch.empty(H, W, 4, **f32), torch.empty(H, W, **f32), torch.empty(H, W, **i32)
    hit_list, hit_count = torch.empty(8 * cap, **i32), torch.empty(16 * T + 2, **i32)
    _lib.check(L.gb_rasterize_ranked_fwd_sort_lists(H, W, 4, p(bins), p(order), p(depths), p(bucket), p(ranks),
                                                    p(records), p(bg4), p(out4), p(final_Ts), p(final_idx),
                                                    p(hit_list), p(hit_count), st), "fwd_sort_lists")
    alpha = 1 - final_Ts
    rgb, a_img, depth = torch.empty(3, H, W, **f32), torch.empty(1, H, W, **f32), torch.empty(1, H, W, **f32)
    _lib.check(L.gb_render_finish_fwd(H, W, p(out4), p(alpha), p(rgb), p(a_img), p(depth), st), "finish_fwd")

    g_out4 = torch.empty(H, W, 4, **f32)
    _lib.check(L.gb_render_finish_bwd(H, W, p(alpha), p(sc["g_rgb"] if use_rgb else None),
                                      p(sc["g_depth"] if use_depth else None), p(g_out4), st), "finish_bwd")
    if acc is None:
        acc = (torch.zeros(G, 2, **f32), torch.zeros(G, 3, **f32), torch.zeros(G, 4, **f32), torch.zeros(G, **f32))
        _lib.check(L.gb_rasterize_ranked_bwd_lists(H, W, 4, p(ranks), p(bins), p(hit_list), p(hit_count), p(records),
                                                   p(bg4), p(final_Ts), p(final_idx), p(g_out4), None,
                                                   *map(p, acc), st), "bwd_lists")
    v_xy, v_conic, v_col4, v_opeff = acc
    v_colors, v_opacity, v_comp, v_depth = (torch.empty(G, 3, **f32), torch.empty(G, 1, **f32), torch.empty(G, **f32),
                                            torch.empty(G, **f32))
    _lib.check(L.gb_splat_grad_unpack(G, p(v_col4), p(v_opeff), p(sc["opacity"]), p(comp), p(v_colors), p(v_opacity),
                                      p(v_comp), p(v_depth), st), "grad_unpack")
    g_cov2d, g_cov3d = torch.empty(G, 3, **f32), torch.empty(G, 6, **f32)
    g_mean, g_scale, g_quat = torch.empty(G, 3, **f32), torch.empty(G, 3, **f32), torch.empty(G, 4, **f32)
    _lib.check(L.gb_project_gaussians_bwd(G, p(sc["means3d"]), p(sc["scales"]), 1.0, p(sc["quats"]),
                                          p(sc["viewmat"]), fx, fy, p(cov3d), p(radii), p(conics), p(comp), p(v_xy),
                                          p(v_depth), p(v_conic), p(v_comp), p(g_cov2d), p(g_cov3d), p(g_mean),
                                          p(g_scale), p(g_quat), st), "project_bwd")
    assert int(ovf) == 0
    return dict(rgb=rgb, alpha=a_img, depth=depth, ranks=ranks[:int(n)], final_Ts=final_Ts, final_idx=final_idx,
                bins=bins, hit_list=hit_list, hit_count=hit_count[:8 * T],
                grads=dict(zip(GRADS, (g_mean, g_scale, g_quat, v_opacity, v_colors))))


def _node(sc, use_rgb=True, use_depth=True):
    """The node under test, forward + backward through autograd; inputs as leaves."""
    from goliath_b200.gsplat.fused import blend_finishes_view, render_fused

    leaves = {k: sc[k].detach().clone().requires_grad_() for k in GRADS}
    assert blend_finishes_view(leaves["means3d"].shape[0], sc["cap"])
    rgb, alpha, depth, _ = render_fused(leaves["means3d"], leaves["scales"], 1.0, leaves["quats"], sc["viewmat"],
                                        *sc["intr"], sc["H"], sc["W"], leaves["opacity"], leaves["colors"],
                                        sc["background"], 0.1, sc["cap"], finish=True)
    saved = rgb.grad_fn.saved_tensors
    pairs = [(rgb, sc["g_rgb"])] * use_rgb + [(depth, sc["g_depth"])] * use_depth
    torch.autograd.backward(*map(list, zip(*pairs)))
    n = int((saved[12][:, 1] - saved[12][:, 0]).sum())  # bins
    T = saved[12].shape[0]
    return dict(rgb=rgb.detach(), alpha=alpha, depth=depth.detach(), ranks=saved[17][:n], final_Ts=saved[15],
                final_idx=saved[16], bins=saved[12], hit_list=saved[18], hit_count=saved[19][:8 * T],
                grads={k: v.grad for k, v in leaves.items()})


def _hit_mask(bins, hit_count):
    """The hit-list entries the forward wrote: per tile t and pixel warp w, hit_count[8 t + w] entries from
    8 bins[t, 0] + w (bins[t, 1] - bins[t, 0])."""
    b, c = t2n(bins).astype(np.int64), t2n(hit_count).astype(np.int64)
    start = (8 * b[:, :1] + np.arange(8)[None] * (b[:, 1:] - b[:, :1])).reshape(-1)
    idx = np.repeat(start - np.cumsum(c) + c, c) + np.arange(c.sum())
    return torch.from_numpy(idx).to(bins.device)


def _check(got, ref, color_grad=True):
    for k in ("rgb", "alpha", "depth", "final_Ts"):
        assert torch.equal(got[k].view(torch.int32), ref[k].view(torch.int32)), k
    for k in ("ranks", "final_idx", "bins", "hit_count"):
        assert torch.equal(got[k], ref[k]), k
    m = _hit_mask(ref["bins"], ref["hit_count"])
    assert torch.equal(got["hit_list"][m], ref["hit_list"][m]), "hit_list"
    for k in GRADS:
        r = t2n(ref["grads"][k])
        assert (np.abs(r).max() > 0) == (k != "colors" or color_grad), k  # only rgb carries a colour gradient
        assert_close(t2n(got["grads"][k]), r, rtol=1e-4, atol=1e-5 * float(np.abs(r).max()), frac=0.9999,
                     what="grad " + k)


@pytest.mark.parametrize("G,cam_k", [(300_000, 0), (300_000, 5), (300_001, 3), (1 << 20, 2)])
def test_node_matches_composition(cuda, G, cam_k):
    sc = _scene(cuda, G, cam_k)
    ref = _parent(sc)
    got = _node(sc)
    torch.cuda.synchronize()
    _check(got, ref)


@pytest.mark.parametrize("use_rgb,use_depth", [(True, False), (False, True)])
def test_absent_view_gradient(cuda, use_rgb, use_depth):
    sc = _scene(cuda, 300_000, 1)
    _check(_node(sc, use_rgb, use_depth), _parent(sc, use_rgb, use_depth), color_grad=use_rgb)


def test_per_gaussian_backward_keeps_its_bits(cuda):
    """The one-pass per-Gaussian backward on the accumulator the node's blend backward filled, against
    gb_splat_grad_unpack + gb_project_gaussians_bwd on the same numbers."""
    from goliath_b200.gsplat.fused import _acc_parts, render_fused

    sc = _scene(cuda, 300_001, 4)
    leaves = {k: sc[k].detach().clone().requires_grad_() for k in GRADS}
    rgb, _, depth, _ = render_fused(leaves["means3d"], leaves["scales"], 1.0, leaves["quats"], sc["viewmat"],
                                    *sc["intr"], sc["H"], sc["W"], leaves["opacity"], leaves["colors"],
                                    sc["background"], 0.1, sc["cap"], finish=True)
    acc = rgb.grad_fn.saved_tensors[10]
    torch.autograd.backward([rgb, depth], [sc["g_rgb"], sc["g_depth"]])
    G = sc["means3d"].shape[0]
    v_col4, v_xy, v_conic, v_opeff = (t.contiguous() for t in _acc_parts(acc, G))
    ref = _parent(sc, acc=(v_xy, v_conic, v_col4, v_opeff))
    torch.cuda.synchronize()
    for k in GRADS:
        assert torch.equal(leaves[k].grad.view(torch.int32), ref["grads"][k].view(torch.int32)), k


def test_graph_replay_matches_eager(cuda):
    """The node captured with its backward in a CUDA graph: every replay zeroes the accumulator in the projection
    again and gives the eager view bit for bit and the eager gradients up to the order of the atomic adds."""
    from goliath_b200.gsplat.fused import render_fused

    sc = _scene(cuda, 300_000, 0)
    ref = _parent(sc)
    leaves = {k: sc[k].detach().clone().requires_grad_() for k in GRADS}

    def step():
        for v in leaves.values():
            v.grad = None
        rgb, alpha, depth, _ = render_fused(leaves["means3d"], leaves["scales"], 1.0, leaves["quats"], sc["viewmat"],
                                            *sc["intr"], sc["H"], sc["W"], leaves["opacity"], leaves["colors"],
                                            sc["background"], 0.1, sc["cap"], finish=True)
        torch.autograd.backward([rgb, depth], [sc["g_rgb"], sc["g_depth"]])
        return rgb, alpha, depth

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            step()
    torch.cuda.current_stream().wait_stream(side)
    for v in leaves.values():
        v.grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        rgb, alpha, depth = step()
    for _ in range(2):
        graph.replay()
        torch.cuda.synchronize()
        for k, t in (("rgb", rgb), ("alpha", alpha), ("depth", depth)):
            assert torch.equal(t.detach().view(torch.int32), ref[k].view(torch.int32)), k
        for k in GRADS:
            r = t2n(ref["grads"][k])
            assert_close(t2n(leaves[k].grad), r, rtol=1e-4, atol=1e-5 * float(np.abs(r).max()), frac=0.9999,
                         what="graph grad " + k)


def test_second_backward_through_retained_graph(cuda):
    """backward twice through one forward (retain_graph): the second pass starts from a zeroed accumulator, so both
    give the same gradients."""
    from goliath_b200.gsplat.fused import render_fused

    sc = _scene(cuda, 200_000, 6)
    leaves = {k: sc[k].detach().clone().requires_grad_() for k in GRADS}
    rgb, _, depth, _ = render_fused(leaves["means3d"], leaves["scales"], 1.0, leaves["quats"], sc["viewmat"],
                                    *sc["intr"], sc["H"], sc["W"], leaves["opacity"], leaves["colors"],
                                    sc["background"], 0.1, sc["cap"], finish=True)
    torch.autograd.backward([rgb, depth], [sc["g_rgb"], sc["g_depth"]], retain_graph=True)
    first = {k: v.grad.clone() for k, v in leaves.items()}
    for v in leaves.values():
        v.grad = None
    torch.autograd.backward([rgb, depth], [sc["g_rgb"], sc["g_depth"]])
    for k in GRADS:
        r = t2n(first[k])
        assert_close(t2n(leaves[k].grad), r, rtol=1e-4, atol=1e-5 * float(np.abs(r).max()), frac=0.9999, what=k)
