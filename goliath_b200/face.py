"""`FaceDecoderFrontal` (ca_code/nn/face.py:16-83), the frozen face decoder that conditions the drivable body avatar's
face region on a face model's latent code, with the reference's constructor, parameter names and shapes, buffer and
Glorot initialisation, so its checkpoints load with strict=True.

With grad disabled (how `mesh_vae_drivable.AutoEncoder` calls it) the first seven `texmod` layers run on the
tensor-core inference path `nn.tower_forward_tc`, and the last layer with its untied bias, the face `bias` and
255 (. + 0.5) on one kernel (`gb_face_tex_tail_fwd`, csrc/body_drive.cu) that writes `face_tex_raw` and `face_tex`.
With grad enabled it composes the differentiable layer kernels and torch's add.  The LinearWN heads are cuBLAS GEMMs.
CUDA only."""
from typing import Dict, Tuple

import numpy as np
import torch
import torch.nn as nn

from . import _lib
from .nn import ConvTranspose2dWNUB, FusedLeakyReLU, LinearWN, _wn_scale, glorot, tower_forward_tc

DEFAULT_TEX_ROI = ((0, 0), (1024, 1024))


def _texmod():
    chans = [(256, 256, 8), (256, 128, 16), (128, 128, 32), (128, 64, 64), (64, 64, 128), (64, 32, 256), (32, 8, 512)]
    layers = []
    for cin, cout, size in chans:
        layer = ConvTranspose2dWNUB(cin, cout, size, size, 4, 2, 1)
        layer.fused_slope = 0.2
        layers += [layer, FusedLeakyReLU()]
    return nn.Sequential(*layers, ConvTranspose2dWNUB(8, 3, 1024, 1024, 4, 2, 1))


def face_tex_tail(x, layer, face_bias):
    """(tex_raw, tex) = (layer(x), 255 (layer(x) + face_bias + 0.5)) for the last texmod layer, forward only"""
    x = x.contiguous()
    _lib.check_input(x, "input")
    B, Cin, Hi, Wi = x.shape
    Cout = layer.out_channels
    v, bias, fb = layer.weight_v.contiguous(), layer.bias.contiguous(), face_bias.contiguous()
    if v.shape != (Cin, Cout, 4, 4) or bias.shape != (Cout, 2 * Hi, 2 * Wi) or fb.shape != bias.shape:
        raise RuntimeError("face texture tail: shapes do not match an input of %s" % (tuple(x.shape),))
    for t, n in ((v, "weight_v"), (bias, "bias"), (fb, "face bias")):
        _lib.check_input(t, n)
    raw = torch.empty(B, Cout, 2 * Hi, 2 * Wi, device=x.device)
    tex = torch.empty_like(raw)
    with torch.cuda.device(x.device):
        _lib.check(_lib.lib().gb_face_tex_tail_fwd(
            B, Cin, Cout, Hi, Wi, _lib.ptr(x), _lib.ptr(v), _lib.ptr(_wn_scale(v, layer.weight_g)), _lib.ptr(bias),
            _lib.ptr(fb), _lib.ptr(raw), _lib.ptr(tex), _lib.stream_ptr(x.device)), "face_tex_tail_fwd")
    return raw, tex


class FaceDecoderFrontal(nn.Module):
    """face.py:16-83.  forward(face_embs [B, n_latent]) -> {face_geom [B, n_vert_out/3, 3], face_tex_raw, face_tex}
    ([B, 3, 1024, 1024]).  Only the default `tex_roi` is accepted: with any other, the reference's `texout + bias`
    does not broadcast."""

    def __init__(self, assets, n_latent: int = 256, n_vert_out: int = 3 * 7306,
                 tex_out_shp: Tuple[int, int] = (1024, 1024), tex_roi=DEFAULT_TEX_ROI) -> None:
        super().__init__()
        if tuple(map(tuple, tex_roi)) != DEFAULT_TEX_ROI:
            raise ValueError("FaceDecoderFrontal: only tex_roi=%s is supported (got %s)" % (DEFAULT_TEX_ROI, tex_roi))
        self.n_latent, self.n_vert_out = n_latent, n_vert_out
        self.tex_roi = tex_roi
        self.tex_roi_shp = tuple(int(i) for i in np.diff(np.array(tex_roi), axis=0).squeeze())
        self.tex_out_shp = tex_out_shp
        self.encmod = nn.Sequential(LinearWN(n_latent, 256), nn.LeakyReLU(0.2, inplace=True))
        self.geommod = nn.Sequential(LinearWN(256, n_vert_out))
        self.viewmod = nn.Sequential(LinearWN(3, 8), nn.LeakyReLU(0.2, inplace=True))
        self.texmod2 = nn.Sequential(LinearWN(256 + 8, 256 * 4 * 4), nn.LeakyReLU(0.2, inplace=True))
        self.texmod = _texmod()
        self.bias = nn.Parameter(torch.zeros(3, self.tex_roi_shp[0], self.tex_roi_shp[1]))
        fv = assets["face_frontal_view"] if isinstance(assets, dict) else assets.face_frontal_view
        self.register_buffer("frontal_view", torch.as_tensor(np.asarray(fv), dtype=torch.float32))
        self.apply(lambda m: glorot(m, 0.2))
        glorot(self.texmod[-1], 1.0)

    def forward(self, face_embs: torch.Tensor) -> Dict[str, torch.Tensor]:
        if not face_embs.is_cuda:
            raise RuntimeError("FaceDecoderFrontal runs on CUDA only (no CPU fallback): face_embs is on %s"
                               % face_embs.device)
        B = face_embs.shape[0]
        view = self.frontal_view[None].expand(B, -1)
        encout = self.encmod(face_embs)
        geomout = self.geommod(encout)
        encview = torch.cat([encout, self.viewmod(view)], dim=1)
        x = self.texmod2(encview).view(-1, 256, 4, 4)
        out = {"face_geom": geomout.view(B, -1, 3)}
        if torch.is_grad_enabled():
            texout = self.texmod(x)
            out["face_tex_raw"] = texout
            out["face_tex"] = 255 * (texout + self.bias[None] + 0.5)
        else:
            x = tower_forward_tc(self.texmod[:-1], x)
            out["face_tex_raw"], out["face_tex"] = face_tex_tail(x, self.texmod[-1], self.bias)
        return out
