"""Drop-in for the reference network class.

`SIGGRAPHGeneratorB200` mirrors `SIGGRAPHGenerator`
(/root/reference/models/pytorch/model.py:5-6 ctor, :134 forward): same constructor, same
`state_dict` keys (so `load_state_dict(torch.load(path))` from
/root/reference/data/colorize_image.py:222-229 works unchanged), same `forward(input_A,
input_B, mask_B, maskcent)` taking numpy [C,X,X] arrays and returning torch tensors that the
wrapper indexes with `[0, :, :, :].cpu().data.numpy()` (:263).  The forward itself runs in
libidc_b200.so; the nn.Module tree below only holds parameters.
"""
import numpy as np
import torch
import torch.nn as nn

from .engine import LhnContext


def _param_tree(mod):
    """Parameter containers with the reference's module names/indices (model.py:13-108).
    ReLU/LeakyReLU/Tanh placeholders keep the Sequential indices identical."""
    def conv(i, o, k=3, d=1):
        return nn.Conv2d(i, o, kernel_size=k, stride=1, padding=d * (k // 2), dilation=d, bias=True)

    def up(i, o):
        return nn.ConvTranspose2d(i, o, kernel_size=4, stride=2, padding=1, bias=True)
    R = lambda: nn.Identity()   # activation slots: computed inside the fused CUDA epilogues
    bn = nn.BatchNorm2d
    mod.model1 = nn.Sequential(conv(4, 64), R(), conv(64, 64), R(), bn(64))
    mod.model2 = nn.Sequential(conv(64, 128), R(), conv(128, 128), R(), bn(128))
    mod.model3 = nn.Sequential(conv(128, 256), R(), conv(256, 256), R(), conv(256, 256), R(), bn(256))
    mod.model4 = nn.Sequential(conv(256, 512), R(), conv(512, 512), R(), conv(512, 512), R(), bn(512))
    mod.model5 = nn.Sequential(conv(512, 512, d=2), R(), conv(512, 512, d=2), R(), conv(512, 512, d=2), R(), bn(512))
    mod.model6 = nn.Sequential(conv(512, 512, d=2), R(), conv(512, 512, d=2), R(), conv(512, 512, d=2), R(), bn(512))
    mod.model7 = nn.Sequential(conv(512, 512), R(), conv(512, 512), R(), conv(512, 512), R(), bn(512))
    mod.model8up = nn.Sequential(up(512, 256))
    mod.model8 = nn.Sequential(R(), conv(256, 256), R(), conv(256, 256), R(), bn(256))
    mod.model9up = nn.Sequential(up(256, 128))
    mod.model9 = nn.Sequential(R(), conv(128, 128), R(), bn(128))
    mod.model10up = nn.Sequential(up(128, 128))
    mod.model10 = nn.Sequential(R(), conv(128, 128), R())
    mod.model3short8 = nn.Sequential(conv(256, 256))
    mod.model2short9 = nn.Sequential(conv(128, 128))
    mod.model1short10 = nn.Sequential(conv(64, 128))
    mod.model_class = nn.Sequential(conv(256, 529, k=1))
    mod.model_out = nn.Sequential(conv(128, 2, k=1), R())


class SIGGRAPHGeneratorB200(nn.Module):
    def __init__(self, dist=False, device=0, engine="wgmma", fast_fp16=False, ref_quirks=True, max_batch=1):
        super(SIGGRAPHGeneratorB200, self).__init__()
        self.dist = dist
        self.b200_device = device
        self.engine = engine
        self.fast_fp16 = fast_fp16
        self.ref_quirks = ref_quirks      # reproduce model.py:166-168 (dist=True returns out_reg*110 again)
        self.max_batch = max_batch
        _param_tree(self)
        for p in self.parameters():
            p.requires_grad_(False)
        self._ctx = {}                    # (H, W, max_n) -> LhnContext
        self._dirty = True
        self.act_ranges = None            # measured activation ranges (set_act_ranges): applied to every context built

    def set_act_ranges(self, ranges):
        """{buffer: max_abs} from engine.measure_act_ranges, or None: ranges belong to the checkpoint, so every
        context this network builds, whatever its geometry, packs its weights with them."""
        self.act_ranges = ranges
        self._dirty = True

    # --- weights: any state change re-packs lazily ---
    def load_state_dict(self, state_dict, strict=True, **kw):
        r = super(SIGGRAPHGeneratorB200, self).load_state_dict(state_dict, strict=strict, **kw)
        self._dirty = True
        return r

    def cuda(self, device=None):
        # reference: `self.net.cuda()` (data/colorize_image.py:230-231).  Parameters stay on the
        # host (they are only the packing source); the packed arena lives on the device.
        if device is not None:
            self.b200_device = device if isinstance(device, int) else torch.device(device).index or 0
            self._ctx = {}
        return self

    def _context(self, H, W, n):
        if self._dirty:
            for c in self._ctx.values():
                c.close()
            self._ctx = {}
            self._dirty = False
        key = (H, W)
        ctx = self._ctx.get(key)
        if ctx is None or ctx.max_n < n:
            if ctx is not None:
                ctx.close()
            ctx = LhnContext(device=self.b200_device, max_n=max(n, self.max_batch), H=H, W=W, dist=self.dist,
                             engine=self.engine, fast_fp16=self.fast_fp16)
            ctx.load_state_dict(self.state_dict(), act_ranges=self.act_ranges)
            self._ctx[key] = ctx
        return ctx

    def forward(self, input_A, input_B, mask_B, maskcent=0):
        """Reference signature (model.py:134): numpy / tensor [1,X,X], [2,X,X], [1,X,X] + float.
        Returns [1,2,X,X] (dist=False) or ([1,2,X,X] * quirk, [1,529,X,X]) (dist=True), as CPU
        torch tensors (the reference's forward also produces CPU tensors, model.py:139-141)."""
        A = np.ascontiguousarray(np.asarray(input_A, dtype=np.float32))[None]
        B = np.ascontiguousarray(np.asarray(input_B, dtype=np.float32))[None]
        M = np.ascontiguousarray(np.asarray(mask_B, dtype=np.float32))[None]
        H, W = A.shape[-2], A.shape[-1]
        ctx = self._context(H, W, 1)
        r = ctx.forward_host(A, B, M, float(maskcent), want_dist=self.dist)
        out_reg = torch.from_numpy(r["ab"])
        if not self.dist:
            return out_reg
        d64 = torch.from_numpy(r["dist"])
        out_cl = d64.repeat_interleave(4, dim=2).repeat_interleave(4, dim=3)   # upsample4, model.py:131,160
        return (out_reg * 110 if self.ref_quirks else out_reg, out_cl)

    def forward_batched(self, L_mc, ab, mask, maskcent=0.0, glob=None, want_dist=None, want_rgb=False):
        """Device tensors [N,1,H,W], [N,2,H,W], [N,1,H,W] -> dict(ab, dist (H/4 grid), rgb)."""
        n, H, W = L_mc.shape[0], L_mc.shape[-2], L_mc.shape[-1]
        ctx = self._context(H, W, n)
        return ctx.forward_device(L_mc, ab, mask, maskcent, glob=glob,
                                  want_dist=self.dist if want_dist is None else want_dist, want_rgb=want_rgb)
