"""Python surface of the SG specular shade with the names and argument meaning of the reference wrapper
(extensions/sgutils/sgutils.py: `EvaluateGaussian` :17-63, `evaluate_gaussian` :65-98), written against the
sm_90a kernels of csrc/sg_shade.cu (through `sgutilslib`).

Contract kept from the reference: lobe directions are normalised in PyTorch so autograd owns that derivative
(:74-75); only lobe_dirs, lobe_sigmas and light_values receive gradients — light_pts, prim_pts and n_lights are
declared non-differentiable (:30); w_type selects one of four lobe shapes (sg.cu:57-70)."""
import torch
import torch.nn.functional as F
from torch.autograd import Function

from . import sgutilslib

_W_TYPES = (0, 1, 2, 3)


def _alloc_like(ref, shape):
    return torch.empty(shape, device=ref.device, dtype=torch.float32)


class EvaluateGaussian(Function):
    """integral[n,d,:] = sum_l light_values[n,l,:] * lobe(angle(lobe_dirs[n,d], light_pts[n,l] - prim_pts[n,d]))."""

    @staticmethod
    def forward(ctx, lobe_dirs, lobe_sigmas, light_values, light_pts, prim_pts, n_lights, w_type):
        if w_type not in _W_TYPES:
            raise AssertionError("w_type must be one of %s" % (_W_TYPES,))
        if light_values.shape[-1] != 3:
            raise AssertionError("light_values must carry 3 channels")
        batch, n_prims = lobe_dirs.shape[0], lobe_dirs.shape[1]
        integral = _alloc_like(lobe_dirs, (batch, n_prims, 3))
        sgutilslib.evaluate_gaussian_fwd(lobe_dirs, lobe_sigmas, light_values, light_pts, prim_pts, n_lights, integral,
                                         w_type)
        ctx.w_type = w_type
        ctx.save_for_backward(lobe_dirs, lobe_sigmas, light_values, light_pts, prim_pts, n_lights)
        ctx.mark_non_differentiable(light_pts, prim_pts, n_lights)
        return integral

    @staticmethod
    def backward(ctx, grad_integral):
        saved = ctx.saved_tensors
        lobe_dirs, lobe_sigmas, light_values = saved[0], saved[1], saved[2]
        # both are fully overwritten by the kernel (the reference zero-fills them first, sgutils.py:43-44)
        d_dirs = _alloc_like(lobe_dirs, lobe_dirs.shape)
        d_sigmas = _alloc_like(lobe_dirs, lobe_sigmas.shape)
        # accumulated with reductions + atomics, hence zero-initialised; only when somebody asks for it
        d_lights = torch.zeros_like(light_values) if ctx.needs_input_grad[2] else None
        sgutilslib.evaluate_gaussian_bwd(*saved, grad_integral.contiguous(), d_dirs, d_sigmas, d_lights, ctx.w_type)
        return d_dirs, d_sigmas, d_lights, None, None, None, None


def _check_shapes(lobe_dirs, lobe_sigmas, light_pts, prim_pts):
    assert lobe_dirs.shape[-1] == 3, lobe_dirs.shape[-1]
    assert lobe_sigmas.dim() == 2 or lobe_sigmas.shape[2] == 1, lobe_sigmas.dim()
    for name, t in (("light_pts", light_pts), ("prim_pts", prim_pts)):
        assert t.dim() == 3 and t.shape[-1] == 3, "%s must be [N, *, 3], got %s" % (name, tuple(t.shape))


def evaluate_gaussian(lobe_dirs, lobe_sigmas, light_values, light_pts, prim_pts, n_lights, w_type: int = 0,
                      normalize_lobe_dirs: bool = True):
    """lobe_dirs [N,D,3], lobe_sigmas [N,D], light_values / light_pts [N,L,3], prim_pts [N,D,3], n_lights [N] int32
    -> integral [N,D,3].  Same call as extensions/sgutils/sgutils.py:65."""
    dirs = F.normalize(lobe_dirs, dim=-1) if normalize_lobe_dirs else lobe_dirs
    _check_shapes(dirs, lobe_sigmas, light_pts, prim_pts)
    return EvaluateGaussian.apply(dirs, lobe_sigmas, light_values, light_pts, prim_pts, n_lights, w_type)
