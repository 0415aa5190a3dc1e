"""fp32 restatement of archs 'basic.HRNet_ASP' and 'mscale.HRNet_ASP' (the ASPP models over the HRNet trunk,
network/basic.py:67-111, network/mscale.py:479-515) assembled from oracle.seg_oracle's HRNet trunk, ASPP, seg head and
attention head, plus the one-step / noise-floor helpers of tests/_parity.py for them. Pinned to the unmodified reference
by tests/golden/reference_hrnet_asp.pt (tests/golden/make_golden_hrnet_asp.py). Test infrastructure only."""
import math
import zlib

import torch

from oracle import seg_oracle as O

ARCHS = ("basic.HRNet_ASP", "mscale.HRNet_ASP")
RED = 256             # cfg.MODEL.ASPP_BOT_CH default (config.py:131)
BOT_CH = 256          # cfg.MODEL.SEGATTN_BOT_CH default (config.py:130)


def _bn_names(name, c):
    return [(name + "." + k, (c,) if k != "num_batches_tracked" else ())
            for k in ("weight", "bias", "running_mean", "running_var", "num_batches_tracked")]


def head_names(arch, high, red=RED, bot=BOT_CH, num_classes=19):
    """(name, shape) of everything after the trunk, in registration order: aspp (features, then img_conv;
    network/utils.py:185-205), bot_aspp, final = make_seg_head(256), and for the mscale model
    scale_attn = make_attn_head(256)."""
    out = [("aspp.features.0.0.weight", (red, high, 1, 1))] + _bn_names("aspp.features.0.1", red)
    for i in range(len(O.ASPP_RATES)):
        out += [("aspp.features.%d.0.weight" % (i + 1), (red, high, 3, 3))] + _bn_names("aspp.features.%d.1" % (i + 1),
                                                                                          red)
    out += [("aspp.img_conv.0.weight", (red, high, 1, 1))] + _bn_names("aspp.img_conv.1", red)
    out += [("bot_aspp.weight", (256, 5 * red, 1, 1))]
    out += [("final.0.weight", (bot, 256, 3, 3))] + _bn_names("final.1", bot)
    out += [("final.3.weight", (bot, bot, 3, 3))] + _bn_names("final.4", bot)
    out += [("final.6.weight", (num_classes, bot, 1, 1))]
    if arch == "mscale.HRNet_ASP":
        out += [("scale_attn.conv0.weight", (bot, 256, 3, 3))] + _bn_names("scale_attn.bn0", bot)
        out += [("scale_attn.conv1.weight", (bot, bot, 3, 3))] + _bn_names("scale_attn.bn1", bot)
        out += [("scale_attn.conv2.weight", (1, bot, 1, 1))]
    return out


def synth_state_dict(arch, hcfg=O.HRNET_W16_TEST, seed=0, red=RED):
    """O.synth_state_dict's deterministic weights (every tensor seeded by crc32(name) ^ seed) for these archs: the trunk
    tensors get the values they have for basic.HRNet. Registration order: backbone, then head_names()."""
    trunk = O.synth_state_dict("basic.HRNet", hcfg, seed=seed)
    sd = {k: v for k, v in trunk.items() if k.startswith("backbone.")}
    for name, shape in head_names(arch, sum(hcfg["stage4"]["num_channels"]), red):
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
        elif name.endswith(".weight"):
            base = name[: -len(".weight")]
            g = torch.Generator().manual_seed((zlib.crc32((base + "#affine").encode()) ^ seed) & 0x7FFFFFFF)
            sd[name] = 1.0 + 0.1 * torch.randn(shape, generator=g)
            sd[base + ".bias"] = 0.1 * torch.randn(shape, generator=g)
    heads = head_names(arch, sum(hcfg["stage4"]["num_channels"]), red)
    order = [k for k in trunk if k.startswith("backbone.")] + [n for n, _s in heads]
    return {k: sd[k] for k in order}


def fwd(ctx, arch, x, hcfg=O.HRNET_W16_TEST):
    """basic.ASPP.forward up to the upsampled logits / mscale.ASPP._fwd (network/basic.py:84-92, network/mscale.py:
    496-511): trunk -> ASPP -> bot_aspp -> seg head (and attention head); both maps upsampled to the pass input size.
    -> (logits, attention or None)."""
    feats = O.hrnet_forward(ctx, "backbone", x, hcfg)
    a = ctx.q(O.conv(ctx, "bot_aspp", O.aspp(ctx, "aspp", feats)))
    cls = O.seg_head(ctx, "final", a)
    attn = O.attn_head(ctx, "scale_attn", a) if arch == "mscale.HRNet_ASP" else None
    size = x.shape[2:]
    return O.bilinear(cls, size), (O.bilinear(attn, size) if attn is not None else None)


def basic_forward(ctx, images, gts=None, criterion=O.criterion_ce, hcfg=O.HRNET_W16_TEST):
    """basic.ASPP.forward (network/basic.py:84-101)."""
    pred, _ = fwd(ctx, "basic.HRNet_ASP", images, hcfg)
    if ctx.training:
        return criterion(pred, gts)
    return dict(pred=pred)


def two_scale(ctx, images, gts=None, criterion=O.criterion_ce, hcfg=O.HRNET_W16_TEST, lo_scale=0.5,
              supervised_mscale_wt=0.0):
    """MscaleBase.two_scale_forward (network/mscale.py:182-220): the 0.5x pass, then the 1.0x pass, whose attention
    map is computed (its BatchNorms update their running statistics) and dropped."""
    pred_05x, attn = fwd(ctx, "mscale.HRNet_ASP", O.resize_x(images, lo_scale), hcfg)
    p_1x, _ = fwd(ctx, "mscale.HRNet_ASP", images, hcfg)
    size = p_1x.shape[2:]
    joint_pred = O.bilinear(attn * pred_05x, size) + (1 - O.bilinear(attn, size)) * p_1x
    if ctx.training:
        loss = criterion(joint_pred, gts)
        if supervised_mscale_wt:
            loss = loss + supervised_mscale_wt * criterion(O.bilinear(pred_05x, size), gts, do_rmi=False)
            loss = loss + supervised_mscale_wt * criterion(p_1x, gts, do_rmi=False)
        return loss
    return dict(pred=joint_pred, pred_05x=pred_05x, pred_10x=p_1x, attn_05x=attn)


def nscale(ctx, images, scales, hcfg=O.HRNET_W16_TEST):
    """MscaleBase.nscale_forward (network/mscale.py:114-180), eval branch."""
    assert 1.0 in scales
    pred = None
    out = {}
    for s in sorted(scales, reverse=True):
        p, attn = fwd(ctx, "mscale.HRNet_ASP", O.resize_x(images, s), hcfg)
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


def forward(ctx, arch, images, gts=None, criterion=O.criterion_ce, hcfg=O.HRNET_W16_TEST, supervised_mscale_wt=0.0):
    """The training loss / evaluation outputs of either arch (two-scale for the mscale model)."""
    if arch == "basic.HRNet_ASP":
        return basic_forward(ctx, images, gts, criterion, hcfg)
    return two_scale(ctx, images, gts, criterion, hcfg, supervised_mscale_wt=supervised_mscale_wt)


# ----------------------------------------------------------------------------------------------- GPU parity helpers
def oracle_train_step(arch, hcfg, sd0, images, gts, sup_wt=0.0, crit=None, emulate_bf16=True, device="cuda"):
    """tests/_parity.py oracle_train_step for these archs: -> (sd with .grad and updated running statistics, loss)."""
    import _parity as P
    P._tf32_off()
    sd = {k: v.clone().to(device) for k, v in sd0.items()}
    for k, v in sd.items():
        if v.is_floating_point() and "running" not in k:
            v.requires_grad_(True)
    ctx = O.Ctx(sd, training=True, emulate_bf16=emulate_bf16)
    loss = forward(ctx, arch, images.to(device), gts.to(device), crit or O.criterion_ce, hcfg, sup_wt)
    loss.backward()
    return sd, float(loss)


def noise_floor(arch, hcfg, sd0, images, gts, sd_ref, sup_wt=0.0, crit=None):
    """tests/_parity.py noise_floor for these archs (the same step on the one-ulp perturbed images)."""
    import _parity as P
    sd_p, _ = oracle_train_step(arch, hcfg, sd0, P.ulp_perturbed(images), gts, sup_wt, crit)
    floor = {name: P.cos_rel(sd_p[name].grad, v.grad) for name, v in sd_ref.items()
             if v.grad is not None and float(v.grad.abs().max()) >= 1e-12}
    run = {k: float((sd_p[k] - v).abs().max() / (v.abs().max() + 1e-6)) for k, v in sd_ref.items()
           if k.endswith("running_mean") or k.endswith("running_var")}
    return floor, run
