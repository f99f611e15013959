"""Drop-in for the reference's pybind module `utilslib` (extensions/utils/utils.cpp:134-137): same function names,
positional arguments and in-place output convention; the kernel is csrc/raydirs.cu on the caller's current stream
(the reference launches on stream 0 with no device guard, utils.cpp:79)."""
from . import _lib


def compute_raydirs_forward(viewposim, viewrotim, focalim, princptim, pixelcoordsim, W, H, volradius, rayposim,
                            raydirim, tminmaxim):
    """utils.cpp:46-82."""
    for t, n in ((viewposim, "viewposim"), (viewrotim, "viewrotim"), (focalim, "focalim"), (princptim, "princptim"),
                 (rayposim, "rayposim"), (raydirim, "raydirim"), (tminmaxim, "tminmaxim")):
        _lib.check_input(t, n)
    if pixelcoordsim is not None:
        _lib.check_input(pixelcoordsim, "pixelcoordsim")
        if pixelcoordsim.size(1) != H or pixelcoordsim.size(2) != W:
            raise RuntimeError("pixelcoordsim must be [N, H, W, 2]")
    N = viewposim.size(0)
    _lib.kernels().gb_compute_raydirs_fwd(
        N, int(H), int(W), viewposim, viewrotim, focalim, princptim, pixelcoordsim, float(volradius), rayposim,
        raydirim, tminmaxim)
    return []


def compute_raydirs_backward(viewposim, viewrotim, focalim, princptim, pixelcoordsim, W, H, volradius, rayposim,
                             raydirim, tminmaxim, grad_viewpos, grad_viewrot, grad_focal, grad_princpt):
    """utils.cpp:84-132: the reference kernel (utils_kernel.cu:53-94) is an empty stub; nothing is written."""
    _lib.kernels().gb_compute_raydirs_bwd()
    return []
