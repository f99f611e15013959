"""Drop-in for the reference's pybind module `sgutilslib` (extensions/sgutils/sg.cu:280-283).

Same function names, positional arguments, in-place output convention (caller allocates, returns [])
and RuntimeError behaviour as the reference binding; the work is done by the sm_90a kernels in
csrc/sg_shade.cu through the C ABI.
"""
import torch

from . import _lib


def _dims(lobe_dirs, light_values):
    return lobe_dirs.size(0), lobe_dirs.size(1), light_values.size(1)


def evaluate_gaussian_fwd(lobe_dirs, lobe_sigmas, light_values, light_pts, prim_pts, n_lights, integral, w_type):
    """sg.cu:177-224.  integral [N,D,3] is written in place."""
    for t, n in ((lobe_dirs, "lobe_dirs"), (lobe_sigmas, "lobe_sigmas"), (light_values, "light_values"),
                 (light_pts, "light_pts"), (prim_pts, "prim_pts"), (integral, "integral")):
        _lib.check_input(t, n)
    _lib.check_input(n_lights, "n_lights", torch.int32)
    N, D, L = _dims(lobe_dirs, light_values)
    for t, n in ((lobe_sigmas, "lobe_sigmas"), (light_values, "light_values"), (light_pts, "light_pts"),
                 (prim_pts, "prim_pts"), (integral, "integral")):
        if t.size(0) != N:
            raise RuntimeError("Batch dim mismatch for %s." % n)
    with torch.cuda.device(lobe_dirs.device):
        _lib.check(_lib.lib().gb_sg_evaluate_fwd(
            _lib.ptr(lobe_dirs), _lib.ptr(lobe_sigmas), _lib.ptr(light_values), _lib.ptr(light_pts),
            _lib.ptr(prim_pts), _lib.ptr(n_lights), _lib.ptr(integral), N, D, L, int(w_type),
            _lib.stream_ptr(lobe_dirs.device)), "evaluate_gaussian_fwd")
    return []


def evaluate_gaussian_bwd(lobe_dirs, lobe_sigmas, light_values, light_pts, prim_pts, n_lights, grad_integral,
                          grad_dirs, grad_lobe_sigmas, grad_light_values, w_type):
    """sg.cu:226-277.  grad_dirs / grad_lobe_sigmas written; grad_light_values (optional) accumulated."""
    for t, n in ((lobe_dirs, "lobe_dirs"), (lobe_sigmas, "lobe_sigmas"), (light_values, "light_values"),
                 (light_pts, "light_pts"), (prim_pts, "prim_pts"), (grad_integral, "grad_integral"),
                 (grad_dirs, "grad_dirs"), (grad_lobe_sigmas, "grad_lobe_sigmas")):
        _lib.check_input(t, n)
    _lib.check_input(n_lights, "n_lights", torch.int32)
    if grad_light_values is not None:
        _lib.check_input(grad_light_values, "grad_light_values")
    N, D, L = _dims(lobe_dirs, light_values)
    with torch.cuda.device(lobe_dirs.device):
        _lib.check(_lib.lib().gb_sg_evaluate_bwd(
            _lib.ptr(lobe_dirs), _lib.ptr(lobe_sigmas), _lib.ptr(light_values), _lib.ptr(light_pts),
            _lib.ptr(prim_pts), _lib.ptr(n_lights), _lib.ptr(grad_integral), _lib.ptr(grad_dirs),
            _lib.ptr(grad_lobe_sigmas), _lib.ptr(grad_light_values), N, D, L, int(w_type),
            _lib.stream_ptr(lobe_dirs.device)), "evaluate_gaussian_bwd")
    return []
