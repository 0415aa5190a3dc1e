"""Architecture description shared by the module constructor and the executor.

``tensor_specs(arch, hcfg, ocfg)`` lists, in the reference's registration order, every parameter/buffer of the
reference module for ``arch`` (names/shapes as in SURVEY.md §8b "State": 1903 keys / 72.14 M parameters for
``ocrnet.HRNet_Mscale``), so checkpoints and optimizer state move between the two implementations by name and
position. Constructors followed: network/hrnetv2.py:263-315 (HighResolutionNet.__init__), network/ocrnet.py:46-83
(OCR_block), network/ocr_utils.py:61-93,129-147, network/utils.py:320-367 (seg / attention heads).
"""

# config.py:161-190 — cfg.MODEL.OCR_EXTRA (HRNetV2-W48)
HRNET_W48 = dict(
    stem=64,
    stage1=dict(num_blocks=[4], num_channels=[64]),
    stage2=dict(num_modules=1, num_blocks=[4, 4], num_channels=[48, 96]),
    stage3=dict(num_modules=4, num_blocks=[4, 4, 4], num_channels=[48, 96, 192]),
    stage4=dict(num_modules=3, num_blocks=[4, 4, 4, 4], num_channels=[48, 96, 192, 384]),
)
# config.py:157-159 (OCR), :130 (SEGATTN_BOT_CH), :131 (ASPP_BOT_CH), network/ocrnet.py:63 (dropout),
# :133-135 (MSCALE_INNER_3x3 / MSCALE_DROPOUT / MSCALE_OLDARCH: --mscale_no3x3 / --mscale_dropout / --mscale_old_arch)
OCR_DEFAULT = dict(mid_channels=512, key_channels=256, num_classes=19, segattn_bot_ch=256, dropout=0.05,
                   aspp_bot_ch=256, mscale_inner_3x3=True, mscale_dropout=False, mscale_oldarch=False)

ARCHS = ("ocrnet.HRNet_Mscale", "ocrnet.HRNet", "basic.HRNet", "mscale.HRNet", "deepv3.DeepV3PlusW38",
         "mscale.DeepV3W38", "basic.HRNet_ASP", "mscale.HRNet_ASP")


def is_two_scale(arch):
    """Architectures whose training forward is the hierarchical two-scale pass (MscaleOCR.two_scale_forward,
    network/ocrnet.py:264-334; MscaleBase.two_scale_forward, network/mscale.py:182-231)."""
    return arch in ("ocrnet.HRNet_Mscale", "mscale.HRNet", "mscale.DeepV3W38", "mscale.HRNet_ASP")


def has_wrn38_trunk(arch):
    """Architectures built on the WideResNet-38 trunk, ASPP and 304-channel decoder (DeepV3Plus, MscaleV3Plus)."""
    return arch in ("deepv3.DeepV3PlusW38", "mscale.DeepV3W38")


def has_hrnet_aspp(arch):
    """Architectures with the ASPP over the HRNet trunk's stride-4 features (basic.ASPP, network/basic.py:67-101;
    mscale.ASPP, network/mscale.py:479-511)."""
    return arch in ("basic.HRNet_ASP", "mscale.HRNet_ASP")


def has_ocr(arch):
    return arch in ("ocrnet.HRNet_Mscale", "ocrnet.HRNet")

# network/wider_resnet.py:303-345 (WiderResNetA2, structure "38", dilation=True) — SURVEY.md §8(f) row f2. Only the
# parameter specification exists so far (checked against the reference's state_dict order); the dilated-convolution /
# pre-activation program is the next row to be built.
WRN38 = dict(structure=[3, 3, 6, 3, 1, 1],
             channels=[(128, 128), (256, 256), (512, 512), (512, 1024), (512, 1024, 2048), (1024, 2048, 4096)])
ASPP_RATES = (12, 24, 36)


def wrn_block_plan(wcfg=WRN38):
    """(module, block, in_ch, channels, stride, dilation, dropout p) per IdentityResidualBlock, forward order."""
    plan, in_ch = [], 64
    for mod_id, num in enumerate(wcfg["structure"]):
        for block_id in range(num):
            dil = 2 if mod_id == 3 else (4 if mod_id > 3 else 1)
            stride = 2 if (block_id == 0 and mod_id == 2) else 1
            drop = 0.3 if mod_id == 4 else (0.5 if mod_id == 5 else None)
            plan.append(("mod%d" % (mod_id + 2), "block%d" % (block_id + 1), in_ch, wcfg["channels"][mod_id], stride,
                         dil, drop))
            in_ch = wcfg["channels"][mod_id][-1]
    return plan


def wrn_drop_layout(wcfg=WRN38):
    """(block prefix, channels of the dropped activation, p) for every bottleneck block that carries a dropout."""
    return [("backbone.%s.%s" % (mod, blk), ch[1], drop) for mod, blk, _i, ch, _s, _d, drop in wrn_block_plan(wcfg)
            if drop is not None and len(ch) == 3]


def aspp_specs(conv, bn, high, red):
    """AtrousSpatialPyramidPoolingModule.__init__ (network/utils.py:174-205): the 1x1 and dilated 3x3 branches
    (`features`), then the image-pooling branch, each `red` (bottleneck_ch) wide over `high` input channels."""
    conv("aspp.features.0.0", red, high, 1); bn("aspp.features.0.1", red)
    for i in range(len(ASPP_RATES)):
        conv("aspp.features.%d.0" % (i + 1), red, high, 3); bn("aspp.features.%d.1" % (i + 1), red)
    conv("aspp.img_conv.0", red, high, 1); bn("aspp.img_conv.1", red)


def attn_head_plan(ocfg, p="scale_attn"):
    """The attention head the cfg selects: ([(conv, bn) of each 3x3 conv + BN + ReLU stage], final 1x1 conv,
    whether nn.Dropout(0.5) sits in front of it).
    make_attn_head (network/utils.py:343-367): conv0/bn0, conv1/bn1 unless MSCALE_INNER_3x3 is off, `drop` when
    MSCALE_DROPOUT is on, conv2. old_make_attn_head (:370-382, MSCALE_OLDARCH, which ignores the other two keys): the
    same two stages and 1x1 conv as an unnamed nn.Sequential (0/1/3/4/6)."""
    if ocfg.get("mscale_oldarch", False):
        return [(p + ".0", p + ".1"), (p + ".3", p + ".4")], p + ".6", False
    stages = [(p + ".conv0", p + ".bn0")]
    if ocfg.get("mscale_inner_3x3", True):
        stages.append((p + ".conv1", p + ".bn1"))
    return stages, p + ".conv2", bool(ocfg.get("mscale_dropout", False))


def attn_head_specs(conv, bn, in_ch, bot, ocfg):
    """Parameters of the attention head over `in_ch` input channels, `bot` (cfg.MODEL.SEGATTN_BOT_CH) wide, in the
    reference's registration order."""
    stages, last, _drop = attn_head_plan(ocfg)
    for i, (c, b) in enumerate(stages):
        conv(c, bot, in_ch if i == 0 else bot, 3); bn(b, bot)
    conv(last, 1, bot, 1)


def deepv3_tensor_specs(num_classes=19, wcfg=WRN38, bot_ch=256, scale_attn=False, ocfg=OCR_DEFAULT):
    """(name, shape, kind) of deepv3.DeepV3PlusW38 in the reference's registration order (network/deepv3.py:46-65,
    network/utils.py:171-202). scale_attn: mscale.DeepV3W38 (MscaleV3Plus.__init__, network/mscale.py:236-277), whose
    decoder `final` is bot_ch (cfg.MODEL.SEGATTN_BOT_CH) wide and is followed by the attention head on the same
    304-channel concat, in the variant ocfg selects (attn_head_plan)."""
    out = []

    def conv(name, o, i, k):
        out.append((name + ".weight", (o, i, k, k), "conv_w"))

    def bn(name, c):
        out.append((name + ".weight", (c,), "bn_w"))
        out.append((name + ".bias", (c,), "bn_b"))
        out.append((name + ".running_mean", (c,), "bn_rm"))
        out.append((name + ".running_var", (c,), "bn_rv"))
        out.append((name + ".num_batches_tracked", (), "bn_nbt"))

    conv("backbone.mod1.conv1", 64, 3, 3)
    for mod, blk, in_ch, ch, stride, _dil, _drop in wrn_block_plan(wcfg):
        b = "backbone.%s.%s" % (mod, blk)
        bn(b + ".bn1.0", in_ch)
        if len(ch) == 2:
            conv(b + ".convs.conv1", ch[0], in_ch, 3); bn(b + ".convs.bn2.0", ch[0])
            conv(b + ".convs.conv2", ch[1], ch[0], 3)
        else:
            conv(b + ".convs.conv1", ch[0], in_ch, 1); bn(b + ".convs.bn2.0", ch[0])
            conv(b + ".convs.conv2", ch[1], ch[0], 3); bn(b + ".convs.bn3.0", ch[1])
            conv(b + ".convs.conv3", ch[2], ch[1], 1)
        if stride != 1 or in_ch != ch[-1]:
            conv(b + ".proj_conv", ch[-1], in_ch, 1)
    high, s2_ch = wcfg["channels"][-1][-1], wcfg["channels"][0][-1]
    aspp_specs(conv, bn, high, 256)
    conv("bot_fine", 48, s2_ch, 1)
    conv("bot_aspp", 256, 256 * (2 + len(ASPP_RATES)), 1)
    conv("final.0", bot_ch, 256 + 48, 3); bn("final.1", bot_ch)
    conv("final.3", bot_ch, bot_ch, 3); bn("final.4", bot_ch)
    conv("final.6", num_classes, bot_ch, 1)
    if scale_attn:      # make_attn_head(304, 1)
        attn_head_specs(conv, bn, 256 + 48, bot_ch, ocfg)
    return out


def hrnet_cfg_from_reference_cfg(cfg):
    """Read the HRNet widths from a reference-style cfg (cfg.MODEL.OCR_EXTRA) when one is importable."""
    ex = cfg.MODEL.OCR_EXTRA
    out = dict(stem=64, stage1=dict(num_blocks=list(ex.STAGE1.NUM_BLOCKS), num_channels=list(ex.STAGE1.NUM_CHANNELS)))
    for key, ref in (("stage2", ex.STAGE2), ("stage3", ex.STAGE3), ("stage4", ex.STAGE4)):
        out[key] = dict(num_modules=ref.NUM_MODULES, num_blocks=list(ref.NUM_BLOCKS),
                        num_channels=list(ref.NUM_CHANNELS))
    return out


def high_level_channels(hcfg):
    return sum(hcfg["stage4"]["num_channels"])


def tensor_specs(arch, hcfg=HRNET_W48, ocfg=OCR_DEFAULT):
    """-> list of (name, shape, kind) with kind in {'conv_w','conv_b','bn_w','bn_b','bn_rm','bn_rv','bn_nbt'}."""
    if arch == "deepv3.DeepV3PlusW38":
        return deepv3_tensor_specs(ocfg["num_classes"], hcfg if "structure" in hcfg else WRN38)
    if arch == "mscale.DeepV3W38":
        return deepv3_tensor_specs(ocfg["num_classes"], hcfg if "structure" in hcfg else WRN38,
                                   ocfg["segattn_bot_ch"], scale_attn=True, ocfg=ocfg)
    out = []

    def conv(name, o, i, k, bias=False):
        out.append((name + ".weight", (o, i, k, k), "conv_w"))
        if bias:
            out.append((name + ".bias", (o,), "conv_b"))

    def bn(name, c):
        out.append((name + ".weight", (c,), "bn_w"))
        out.append((name + ".bias", (c,), "bn_b"))
        out.append((name + ".running_mean", (c,), "bn_rm"))
        out.append((name + ".running_var", (c,), "bn_rv"))
        out.append((name + ".num_batches_tracked", (), "bn_nbt"))

    p = "backbone"
    conv(p + ".conv1", 64, 3, 3); bn(p + ".bn1", 64)
    conv(p + ".conv2", 64, 64, 3); bn(p + ".bn2", 64)
    s1 = hcfg["stage1"]
    planes, inpl = s1["num_channels"][0], hcfg["stem"]
    for k in range(s1["num_blocks"][0]):
        b = "%s.layer1.%d" % (p, k)
        conv(b + ".conv1", planes, inpl, 1); bn(b + ".bn1", planes)
        conv(b + ".conv2", planes, planes, 3); bn(b + ".bn2", planes)
        conv(b + ".conv3", planes * 4, planes, 1); bn(b + ".bn3", planes * 4)
        if k == 0 and inpl != planes * 4:
            conv(b + ".downsample.0", planes * 4, inpl, 1); bn(b + ".downsample.1", planes * 4)
        inpl = planes * 4
    pre = [planes * 4]
    for si, key in ((1, "stage2"), (2, "stage3"), (3, "stage4")):
        sc = hcfg[key]
        ch = sc["num_channels"]
        tp = "%s.transition%d" % (p, si)
        for i in range(len(ch)):
            if i < len(pre):
                if ch[i] != pre[i]:
                    conv("%s.%d.0" % (tp, i), ch[i], pre[i], 3); bn("%s.%d.1" % (tp, i), ch[i])
            else:
                for j in range(i + 1 - len(pre)):
                    oc = ch[i] if j == i - len(pre) else pre[-1]
                    conv("%s.%d.%d.0" % (tp, i, j), oc, pre[-1], 3); bn("%s.%d.%d.1" % (tp, i, j), oc)
        nb = len(ch)
        for m in range(sc["num_modules"]):
            mp = "%s.%s.%d" % (p, key, m)
            for i in range(nb):
                for k in range(sc["num_blocks"][i]):
                    b = "%s.branches.%d.%d" % (mp, i, k)
                    conv(b + ".conv1", ch[i], ch[i], 3); bn(b + ".bn1", ch[i])
                    conv(b + ".conv2", ch[i], ch[i], 3); bn(b + ".bn2", ch[i])
            for i in range(nb):
                for j in range(nb):
                    fp = "%s.fuse_layers.%d.%d" % (mp, i, j)
                    if j > i:
                        conv(fp + ".0", ch[i], ch[j], 1); bn(fp + ".1", ch[i])
                    elif j < i:
                        for k in range(i - j):
                            oc = ch[i] if k == i - j - 1 else ch[j]
                            conv("%s.%d.0" % (fp, k), oc, ch[j], 3); bn("%s.%d.1" % (fp, k), oc)
        pre = ch
    high = sum(pre)
    if arch in ("ocrnet.HRNet", "ocrnet.HRNet_Mscale"):
        mid, key_ch, ncls = ocfg["mid_channels"], ocfg["key_channels"], ocfg["num_classes"]
        o = "ocr"
        conv(o + ".conv3x3_ocr.0", mid, high, 3, True); bn(o + ".conv3x3_ocr.1.0", mid)
        ob = o + ".ocr_distri_head.object_context_block"
        conv(ob + ".f_pixel.0", key_ch, mid, 1); bn(ob + ".f_pixel.1.0", key_ch)
        conv(ob + ".f_pixel.2", key_ch, key_ch, 1); bn(ob + ".f_pixel.3.0", key_ch)
        conv(ob + ".f_object.0", key_ch, mid, 1); bn(ob + ".f_object.1.0", key_ch)
        conv(ob + ".f_object.2", key_ch, key_ch, 1); bn(ob + ".f_object.3.0", key_ch)
        conv(ob + ".f_down.0", key_ch, mid, 1); bn(ob + ".f_down.1.0", key_ch)
        conv(ob + ".f_up.0", mid, key_ch, 1); bn(ob + ".f_up.1.0", mid)
        cb = o + ".ocr_distri_head.conv_bn_dropout"
        conv(cb + ".0", mid, 2 * mid, 1); bn(cb + ".1.0", mid)
        conv(o + ".cls_head", ncls, mid, 1, True)
        conv(o + ".aux_head.0", high, high, 1, True); bn(o + ".aux_head.1.0", high)
        conv(o + ".aux_head.2", ncls, high, 1, True)
        if arch == "ocrnet.HRNet_Mscale":
            attn_head_specs(conv, bn, mid, ocfg["segattn_bot_ch"], ocfg)
    elif arch == "basic.HRNet":
        bot, ncls = ocfg["segattn_bot_ch"], ocfg["num_classes"]
        s = "seg_head"
        conv(s + ".0", bot, high, 3); bn(s + ".1", bot)
        conv(s + ".3", bot, bot, 3); bn(s + ".4", bot)
        conv(s + ".6", ncls, bot, 1)
    elif has_hrnet_aspp(arch):
        # basic.ASPP / mscale.ASPP.__init__ (network/basic.py:71-82, network/mscale.py:483-494): get_aspp(720,
        # ASPP_BOT_CH) -> bot_aspp (1x1 to 256, no bias) -> final = make_seg_head(256) [-> scale_attn =
        # make_attn_head(256)]
        red, bot, ncls = ocfg["aspp_bot_ch"], ocfg["segattn_bot_ch"], ocfg["num_classes"]
        aspp_specs(conv, bn, high, red)
        conv("bot_aspp", 256, red * (2 + len(ASPP_RATES)), 1)
        conv("final.0", bot, 256, 3); bn("final.1", bot)
        conv("final.3", bot, bot, 3); bn("final.4", bot)
        conv("final.6", ncls, bot, 1)
        if arch == "mscale.HRNet_ASP":
            attn_head_specs(conv, bn, 256, bot, ocfg)
    elif arch == "mscale.HRNet":
        # MscaleBasic.__init__ (network/mscale.py:450-461): backbone, cls_head = make_seg_head, scale_attn = make_attn_head
        bot, ncls = ocfg["segattn_bot_ch"], ocfg["num_classes"]
        s = "cls_head"
        conv(s + ".0", bot, high, 3); bn(s + ".1", bot)
        conv(s + ".3", bot, bot, 3); bn(s + ".4", bot)
        conv(s + ".6", ncls, bot, 1)
        attn_head_specs(conv, bn, high, bot, ocfg)
    else:
        raise ValueError("unsupported arch %r (hot path covers %s)" % (arch, ", ".join(ARCHS)))
    return out
