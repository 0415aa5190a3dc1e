"""fp32 restatement of arch 'mscale.DeepV3W38' (MscaleV3Plus over the WideResNet-38 trunk, network/mscale.py:232-336)
assembled from oracle.seg_oracle's WRN-38 / ASPP / decoder pieces and its attention head, plus the one-step / noise-floor
helpers of tests/_parity.py for it. Pinned to the unmodified reference by tests/golden/reference_mscale_deepv3.pt
(tests/golden/make_golden_mscale_deepv3.py). Test infrastructure only."""
import math
import zlib

import torch
import torch.nn.functional as F

from oracle import seg_oracle as O

ARCH = "mscale.DeepV3W38"
BOT_CH = 256          # cfg.MODEL.SEGATTN_BOT_CH default (config.py:130)


def _attn_names(bot=BOT_CH):
    """scale_attn = make_attn_head(304, 1) (network/utils.py:343-367), registered after `final`."""
    out = [("scale_attn.conv0.weight", (bot, 256 + 48, 3, 3))]
    out += [("scale_attn.bn0." + k, (bot,) if k != "num_batches_tracked" else ())
            for k in ("weight", "bias", "running_mean", "running_var", "num_batches_tracked")]
    out += [("scale_attn.conv1.weight", (bot, bot, 3, 3))]
    out += [("scale_attn.bn1." + k, (bot,) if k != "num_batches_tracked" else ())
            for k in ("weight", "bias", "running_mean", "running_var", "num_batches_tracked")]
    out += [("scale_attn.conv2.weight", (1, bot, 1, 1))]
    return out


def state_dict_names(wcfg=O.WRN38, num_classes=19):
    """(name, shape) of MscaleV3Plus's state_dict in registration order: backbone, aspp, bot_fine, bot_aspp, final,
    scale_attn (network/mscale.py:242-277)."""
    return O._deepv3_names(wcfg, num_classes) + _attn_names()


def synth_state_dict(wcfg=O.WRN38, seed=0):
    """O.synth_state_dict's deterministic weights (every tensor seeded by crc32(name) ^ seed) for this arch: the tensors
    it shares with deepv3.DeepV3PlusW38 get the same values."""
    sd = O.synth_state_dict("deepv3.DeepV3PlusW38", wcfg, seed=seed)
    for name, shape in _attn_names():
        if name.endswith("num_batches_tracked"):
            sd[name] = torch.zeros((), dtype=torch.long)
        elif name.endswith("running_mean"):
            sd[name] = torch.zeros(shape)
        elif name.endswith("running_var"):
            sd[name] = torch.ones(shape)
        elif len(shape) == 4:
            g = torch.Generator().manual_seed((zlib.crc32(name.encode()) ^ seed) & 0x7FFFFFFF)
            fan_in = shape[1] * shape[2] * shape[3]
            sd[name] = torch.randn(shape, generator=g) * math.sqrt(2.0 / fan_in)
    for base in ("scale_attn.bn0", "scale_attn.bn1"):
        g = torch.Generator().manual_seed((zlib.crc32((base + "#affine").encode()) ^ seed) & 0x7FFFFFFF)
        c = sd[base + ".running_mean"].shape[0]
        sd[base + ".weight"] = 1.0 + 0.1 * torch.randn(c, generator=g)
        sd[base + ".bias"] = 0.1 * torch.randn(c, generator=g)
    return {name: sd[name] for name, _s in state_dict_names(wcfg)}


def fwd(ctx, x, wcfg=O.WRN38):
    """MscaleV3Plus._fwd (network/mscale.py:296-328) with fuse_aspp and attn_2b off: the decoder `final` and the
    attention head both read [bot_fine(s2) | up(bot_aspp(aspp))]; both maps are upsampled to the pass input size."""
    q = ctx.q
    s2, _s4, final = O.wrn38_forward(ctx, "backbone", q(x), wcfg)     # the product reads the image as bf16
    conv_aspp = q(O.conv(ctx, "bot_aspp", O.aspp(ctx, "aspp", final)))
    conv_s2 = q(O.conv(ctx, "bot_fine", s2))
    cat = torch.cat([conv_s2, O.bilinear(conv_aspp, s2.shape[2:])], 1)
    t = q(F.relu(O.bn(ctx, "final.1", q(O.conv(ctx, "final.0", cat, 1, 1)))))
    t = q(F.relu(O.bn(ctx, "final.4", q(O.conv(ctx, "final.3", t, 1, 1)))))
    cls = ctx.qg(O.conv(ctx, "final.6", t))
    attn = O.attn_head(ctx, "scale_attn", cat)
    size = x.shape[2:]
    return O.bilinear(cls, size), O.bilinear(attn, size)


def two_scale(ctx, images, gts=None, criterion=O.criterion_ce, wcfg=O.WRN38, lo_scale=0.5, supervised_mscale_wt=0.0):
    """MscaleBase.two_scale_forward (network/mscale.py:182-220): the 0.5x pass first (its Dropout2d masks are drawn
    first), then the 1.0x pass, whose attention map is computed and dropped."""
    pred_05x, attn = fwd(ctx, O.resize_x(images, lo_scale), wcfg)
    p_1x, _ = fwd(ctx, images, wcfg)
    size = p_1x.shape[2:]
    joint_pred = O.bilinear(attn * pred_05x, size) + (1 - O.bilinear(attn, size)) * p_1x
    if ctx.training:
        loss = criterion(joint_pred, gts)
        if supervised_mscale_wt:
            loss = loss + supervised_mscale_wt * criterion(O.bilinear(pred_05x, size), gts, do_rmi=False)
            loss = loss + supervised_mscale_wt * criterion(p_1x, gts, do_rmi=False)
        return loss
    return dict(pred=joint_pred, pred_05x=pred_05x, pred_10x=p_1x, attn_05x=attn)


def nscale(ctx, images, scales, wcfg=O.WRN38):
    """MscaleBase.nscale_forward (network/mscale.py:114-180), eval branch."""
    assert 1.0 in scales
    pred = None
    out = {}
    for s in sorted(scales, reverse=True):
        p, attn = fwd(ctx, O.resize_x(images, s), wcfg)
        out[O.fmt_scale("pred", s)] = p
        if s != 2.0:
            out[O.fmt_scale("attn", s)] = attn
        if pred is None:
            pred = p
        elif s >= 1.0:
            pred = attn * p + (1 - attn) * O.bilinear(pred, p.shape[2:])
        else:
            p = O.bilinear(attn * p, pred.shape[2:])
            attn = O.bilinear(attn, pred.shape[2:])
            pred = p + (1 - attn) * pred
    out["pred"] = pred
    return out


# ----------------------------------------------------------------------------------------------- GPU parity helpers
def mask_fn(keep_masks):
    """Ctx.drop_mask_fn replaying 0/1 keep masks ([n, c] each) in the order the Dropout2d layers run."""
    it = iter(keep_masks)

    def fn(shape):
        m = next(it)
        assert tuple(m.shape) == tuple(shape[:2]), (m.shape, shape)
        return m.view(shape)
    return fn


def oracle_train_step(wcfg, sd0, images, gts, keep_masks=None, sup_wt=0.0, crit=None, emulate_bf16=True, device="cuda"):
    """tests/_parity.py oracle_train_step for this arch: -> (sd with .grad and updated running statistics, loss)."""
    import _parity as P
    P._tf32_off()
    sd = {k: v.clone().to(device) for k, v in sd0.items()}
    for k, v in sd.items():
        if v.is_floating_point() and "running" not in k:
            v.requires_grad_(True)
    ctx = O.Ctx(sd, training=True, emulate_bf16=emulate_bf16,
                drop_mask_fn=mask_fn([m.to(device) for m in keep_masks]) if keep_masks is not None else None)
    loss = two_scale(ctx, images.to(device), gts.to(device), criterion=crit or O.criterion_ce, wcfg=wcfg,
                     supervised_mscale_wt=sup_wt)
    loss.backward()
    return sd, float(loss)


def noise_floor(wcfg, sd0, images, gts, sd_ref, keep_masks=None, sup_wt=0.0, crit=None):
    """tests/_parity.py noise_floor for this arch (the same masks on the one-ulp perturbed images)."""
    import _parity as P
    sd_p, _ = oracle_train_step(wcfg, sd0, P.ulp_perturbed(images), gts, keep_masks, sup_wt, crit)
    floor = {name: P.cos_rel(sd_p[name].grad, v.grad) for name, v in sd_ref.items()
             if v.grad is not None and float(v.grad.abs().max()) >= 1e-12}
    run = {k: float((sd_p[k] - v).abs().max() / (v.abs().max() + 1e-6)) for k, v in sd_ref.items()
           if k.endswith("running_mean") or k.endswith("running_var")}
    return floor, run
