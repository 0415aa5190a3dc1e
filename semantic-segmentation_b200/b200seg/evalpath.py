"""Eval-mode forward: per-scale passes on the sm_90a kernels (BatchNorm from running statistics, no tape), then the
reference's output assembly in fp32 NCHW on the device.

  ocrnet.HRNet_Mscale : MscaleOCR.nscale_forward when cfg.MODEL.N_SCALES is set (network/ocrnet.py:185-262), else the
                        eval branch of two_scale_forward (:264-327)
  mscale.HRNet        : MscaleBase.nscale_forward / two_scale_forward eval branches (network/mscale.py:114-231)
  ocrnet.HRNet        : OCRNet.forward eval branch (:104-122)
  basic.HRNet         : Basic.forward eval branch (network/basic.py:50-64)
  deepv3.DeepV3PlusW38: DeepV3Plus.forward eval branch (network/deepv3.py:73-96)
"""
import torch

from . import arch as A
from . import model as M
from . import raw
from .engine import Engine


def _fmt_scale(prefix, scale):
    """utils/misc.fmt_scale (utils/misc.py:503-513): keeps the dot ('pred_0.5x')."""
    return "%s_%sx" % (prefix, str(float(scale)))


def _pass(module, E, images, size_hw):
    """One scale pass -> full-resolution (= pass input size) fp32 NCHW cls / aux / attn maps (MscaleOCR._fwd)."""
    out = M.scale_pass(E, images, size_hw, module.arch, module.hcfg, module.ocfg)
    H, W = size_hw
    res = dict(cls_out=raw.resize_to_nchw(out["cls"].logits, 19, H, W))
    # the full-resolution auxiliary map only feeds the training loss (network/ocrnet.py:254-259): dead in eval mode
    if out["attn"] is not None:
        res["logit_attn"] = raw.resize_to_nchw(out["attn"].logits, 1, H, W, apply_sigmoid=True)
    return res


@torch.no_grad()
def eval_forward(module, images):
    module._ensure_device_state()
    module._repack()
    images = images.contiguous().float()
    n, _, H, W = images.shape
    tensors = {k: v.detach() for k, v in module._tensors().items()}
    E = Engine(tensors, {}, module._packed, False, None)
    # BatchNorm from running statistics: every layer's scale / shift up front; conv + BN (+ residual) + ReLU then run as
    # ONE launch each (raw.conv2d_fwd_affine). B200SEG_EVAL_FUSED=0: separate bn_eval_params / bn_apply launches.
    import os
    if os.environ.get("B200SEG_EVAL_FUSED", "1") == "1":
        E.eval_bn = module._eval_bn_params()
    arch = module.arch
    if arch == "deepv3.DeepV3PlusW38":          # DeepV3Plus.forward eval branch (network/deepv3.py:73-96)
        head = M.deepv3_pass(E, images, module.hcfg)
        return {"pred": raw.resize_to_nchw(head.logits, 19, H, W)}
    if not A.is_two_scale(arch):
        return {"pred": _pass(module, E, images, (H, W))["cls_out"]}

    if module.n_scales:
        scales = sorted([float(s) for s in module.n_scales], reverse=True)
        assert 1.0 in scales, "expected 1.0 to be the target scale"
        pred = None
        out = {}
        for s in scales:
            hs, ws = int(H * s), int(W * s)             # ResizeX: floor(in * scale)
            o = _pass(module, E, images, (hs, ws))
            cls, attn = o["cls_out"], o["logit_attn"]
            out[_fmt_scale("pred", s)] = cls
            if s != 2.0:
                out[_fmt_scale("attn", s)] = attn
            if pred is None:
                pred = cls
            elif s >= 1.0:
                pred = raw.blend(attn, cls, raw.resize_nchw(pred, hs, ws), 0)
            else:
                ph, pw = pred.shape[2:]
                cls_s = raw.resize_nchw(raw.blend(attn, cls, None, 2), ph, pw)
                attn_s = raw.resize_nchw(attn, ph, pw)
                pred = raw.blend(attn_s, cls_s, pred, 1)
        out["pred"] = pred
        return out

    hm, wm = int(H * module.lo_scale), int(W * module.lo_scale)
    lo = _pass(module, E, images, (hm, wm))
    hi = _pass(module, E, images, (H, W))
    attn = lo["logit_attn"]
    p_lo = raw.resize_nchw(raw.blend(attn, lo["cls_out"], None, 2), H, W)
    attn_up = raw.resize_nchw(attn, H, W)
    joint = raw.blend(attn_up, p_lo, hi["cls_out"], 1)
    return {"pred": joint, "pred_05x": lo["cls_out"], "pred_10x": hi["cls_out"], "attn_05x": attn}
