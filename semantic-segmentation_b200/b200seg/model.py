"""Network programs for the executor: HRNetV2 backbone, OCR head, attention head, multi-scale loss.

Each function mirrors one reference forward (cited), expressed with ``Engine`` fused ops on NHWC bf16 activations.
"""
import torch

from . import arch as A
from . import raw
from .engine import Act, BF16, F32


# ----------------------------------------------------------------------------------------------- backbone
def basic_block(E, p, x):
    """hrnetv2.BasicBlock.forward (network/hrnetv2.py:50-66)."""
    t = E.conv_bn(x, p + ".conv1", p + ".bn1", 3, relu=True)
    return E.conv_bn(t, p + ".conv2", p + ".bn2", 3, relu=True, residual=x)


def bottleneck(E, p, x, has_downsample):
    """hrnetv2.Bottleneck.forward (network/hrnetv2.py:86-106)."""
    t = E.conv_bn(x, p + ".conv1", p + ".bn1", 1, relu=True)
    t = E.conv_bn(t, p + ".conv2", p + ".bn2", 3, relu=True)
    rec = E.conv_stats(t, p + ".conv3", p + ".bn3", 1)
    if has_downsample:
        ds = E.conv_stats(x, p + ".downsample.0", p + ".downsample.1", 1)
        n, h, w, c = rec.y.shape
        return E.fuse((n, h, w, c), [("rec", rec), ("rec", ds)], relu=True)   # out = relu(bn3(.) + bn_ds(.))
    return E.bn_act(rec, relu=True, residual=x)


def hr_module(E, p, xs, num_blocks, out0=None):
    """HighResolutionModule.forward (network/hrnetv2.py:230-254). out0: optional view for the branch-0 output."""
    nb = len(xs)
    xs = list(xs)
    E.fork(nb)                       # the branches are independent: parallel streams / graph branches
    for i in range(nb):
        with E.on_branch(i):
            for k in range(num_blocks[i]):
                xs[i] = basic_block(E, "%s.branches.%d.%d" % (p, i, k), xs[i])
    E.join(nb)
    outs = []
    for i in range(nb):
        terms = []
        for j in range(nb):
            fp = "%s.fuse_layers.%d.%d" % (p, i, j)
            if j == i:
                terms.append(("id", xs[j]))
            elif j > i:
                terms.append(("rec", E.conv_stats(xs[j], fp + ".0", fp + ".1", 1)))
            else:
                t = xs[j]
                for k in range(i - j - 1):
                    t = E.conv_bn(t, "%s.%d.0" % (fp, k), "%s.%d.1" % (fp, k), 3, stride=2, relu=True)
                k = i - j - 1
                terms.append(("rec", E.conv_stats(t, "%s.%d.0" % (fp, k), "%s.%d.1" % (fp, k), 3, stride=2)))
        outs.append(E.fuse(tuple(xs[i].t.shape), terms, relu=True, out=out0 if i == 0 else None))
    return outs


def hrnet_forward(E, x16, hcfg, p="backbone"):
    """HighResolutionNet.forward (network/hrnetv2.py:399-449) on the 16-channel-padded bf16 image.
    Returns the concatenated 1/4-resolution feature Act [N, H/4, W/4, sum(C)]."""
    x = E.conv_bn(x16, p + ".conv1", p + ".bn1", 3, stride=2, relu=True)
    x = E.conv_bn(x, p + ".conv2", p + ".bn2", 3, stride=2, relu=True)
    s1 = hcfg["stage1"]
    for k in range(s1["num_blocks"][0]):
        x = bottleneck(E, "%s.layer1.%d" % (p, k), x, k == 0 and s1["num_channels"][0] * 4 != hcfg["stem"])
    pre = [s1["num_channels"][0] * 4]
    ys = [x]
    cat = None
    for si, key in ((1, "stage2"), (2, "stage3"), (3, "stage4")):
        sc = hcfg[key]
        ch = sc["num_channels"]
        tp = "%s.transition%d" % (p, si)
        xs = []
        for i in range(len(ch)):
            if i < len(pre):
                if ch[i] != pre[i]:
                    xs.append(E.conv_bn(ys[i], "%s.%d.0" % (tp, i), "%s.%d.1" % (tp, i), 3, relu=True))
                else:
                    xs.append(ys[i])
            else:
                t = ys[-1]
                for j in range(i + 1 - len(pre)):
                    t = E.conv_bn(t, "%s.%d.%d.0" % (tp, i, j), "%s.%d.%d.1" % (tp, i, j), 3, stride=2, relu=True)
                xs.append(t)
        for m in range(sc["num_modules"]):
            out0 = None
            if key == "stage4" and m == sc["num_modules"] - 1:
                # final module: branch 0 is written straight into the concat buffer (network/hrnetv2.py:438-447)
                n, h, w, _ = xs[0].t.shape
                cat = Act(raw._new((n, h, w, sum(ch)), dtype=BF16, device=xs[0].t.device))
                out0 = cat.t[..., : ch[0]]
            xs = hr_module(E, "%s.%s.%d" % (p, key, m), xs, sc["num_blocks"], out0=out0)
        ys = xs
        pre = ch
    # upsample branches 1.. into their channel slices of the concat buffer
    n, h, w, ctot = cat.t.shape
    pieces = [(ys[0], 0, pre[0])]
    c0 = pre[0]
    for j in range(1, len(ys)):
        view = cat.t[..., c0:c0 + pre[j]]
        up = E.fuse((n, h, w, pre[j]), [("id", ys[j])], relu=False, out=view)
        pieces.append((up, c0, c0 + pre[j]))
        c0 += pre[j]
    E.slice_marker(cat, pieces)
    return cat


# ----------------------------------------------------------------------------------------------- OCR head
def spatial_gather(E, feats, aux, K):
    """SpatialGather_Module.forward (network/ocr_utils.py:34-46): context[n,k,:] = sum_pix softmax_pix(aux)[pix,k] *
    feats[pix,:]. The softmax runs over pixels; the product is the wgmma weight-gradient GEMM (pixels = reduction).
    feats: Act [n,h,w,C]; aux: HeadRec with fp32 logits. Returns the proxy Act [n,K,1,C] (bf16)."""
    n, h, w, C = feats.t.shape
    P = h * w
    dev = feats.t.device
    ld = aux.logits.stride(2)
    probs = raw.spatial_softmax_fwd(aux.logits.as_strided((n, P, ld), (P * ld, ld, 1)), K)     # [n,P,32] bf16
    ctx32 = raw._newz((n, K, C), dtype=F32, device=dev)
    for i in range(n):
        raw.conv2d_wgrad(feats.t[i:i + 1], probs[i].view(1, h, w, 32), ctx32[i].view(K, C, 1, 1), K, 1, 1)
    proxy = Act(raw._new((n, K, 1, C), dtype=BF16, device=dev))
    raw.cast_rows(ctx32.view(n * K, C), proxy.t.view(n * K, C), C)

    def gather_bwd():
        if proxy.grad is None:
            return
        dprob = raw._new((n, P, 20), dtype=F32, device=dev)
        if feats.grad is None:
            feats.grad = raw._newz(feats.t.shape, dtype=BF16, device=dev)
        for i in range(n):
            dctx = proxy.grad[i].view(K, C)                         # bf16 [K, C]
            raw.conv2d_fwd(feats.t[i:i + 1], dctx.view(K, 1, C), out_fp32=True,
                           out=dprob[i].view(1, h, w, 20)[..., :K])
            wT = raw.transpose_pad(dctx, 24).view(C, 1, 24)         # [C][1][24]
            raw.conv2d_dgrad(probs[i].view(1, h, w, 32)[..., :24], wT, (1, h, w, C), 1, 1,
                             addend=feats.grad[i:i + 1], out=feats.grad[i:i + 1])
        if aux.dlogits is None:
            aux.dlogits = raw._newz((n, h, w, 32), dtype=BF16, device=dev)
        raw.spatial_softmax_bwd(dprob, probs, K, aux.dlogits.view(n, P, 32), True)
        proxy.grad = None
    E._push(gather_bwd)
    return proxy


def object_attention(E, q, kk, vv, K):
    """Core of ObjectAttentionBlock.forward (network/ocr_utils.py:100-113): sim = softmax_k(q . k / sqrt(C)),
    context = sim . v. q: Act [n,h,w,C]; kk, vv: Acts [n,K,1,C] (f_object / f_down outputs). Returns Act [n,h,w,C]."""
    n, h, w, C = q.t.shape
    P = h * w
    dev = q.t.device
    scale = float(C) ** -0.5
    ctx = Act(raw._new((n, h, w, C), dtype=BF16, device=dev))
    sims = []
    for i in range(n):
        kmat = kk.t[i].view(K, 1, C)
        sl = raw.conv2d_fwd(q.t[i:i + 1], kmat, out_fp32=True, out_ld=20)              # [1,h,w,K] fp32
        sim = raw.class_softmax_fwd(sl.as_strided((P, 20), (20, 1)), K, scale)         # [P,32] bf16
        sims.append(sim)
        vT = raw.transpose_pad(vv.t[i].view(K, C), 24).view(C, 1, 24)
        raw.conv2d_dgrad(sim.view(1, h, w, 32)[..., :24], vT, (1, h, w, C), 1, 1, out=ctx.t[i:i + 1])

    def attend_bwd():
        dctx = ctx.grad
        if dctx is None:
            return
        if q.grad is None:
            q.grad = raw._newz(q.t.shape, dtype=BF16, device=dev)
        if kk.grad is None:
            kk.grad = raw._newz(kk.t.shape, dtype=BF16, device=dev)
        if vv.grad is None:
            vv.grad = raw._newz(vv.t.shape, dtype=BF16, device=dev)
        for i in range(n):
            sim = sims[i]
            vmat = vv.t[i].view(K, 1, C)
            dsim = raw.conv2d_fwd(dctx[i:i + 1], vmat, out_fp32=True, out_ld=20)
            ds = raw.class_softmax_bwd(dsim.as_strided((P, 20), (20, 1)), sim, K, scale)     # [P,32] bf16
            kT = raw.transpose_pad(kk.t[i].view(K, C), 24).view(C, 1, 24)
            raw.conv2d_dgrad(ds.view(1, h, w, 32)[..., :24], kT, (1, h, w, C), 1, 1, addend=q.grad[i:i + 1],
                             out=q.grad[i:i + 1])
            dk = raw._newz((K, C), dtype=F32, device=dev)
            raw.conv2d_wgrad(q.t[i:i + 1], ds.view(1, h, w, 32), dk.view(K, C, 1, 1), K, 1, 1)
            raw.cast_rows(dk, kk.grad[i].view(K, C), C, accumulate=True)
            dv = raw._newz((K, C), dtype=F32, device=dev)
            raw.conv2d_wgrad(dctx[i:i + 1], sim.view(1, h, w, 32), dv.view(K, C, 1, 1), K, 1, 1)
            raw.cast_rows(dv, vv.grad[i].view(K, C), C, accumulate=True)
        ctx.grad = None
    E._push(attend_bwd)
    return ctx


def ocr_block(E, feats_in, ocfg, p="ocr"):
    """OCR_block.forward (network/ocrnet.py:85-91) + SpatialOCR_Module.forward (network/ocr_utils.py:149-158).
    Returns (cls HeadRec, aux HeadRec, ocr_feats Act)."""
    mid, K = ocfg["mid_channels"], ocfg["num_classes"]
    n, h, w, _ = feats_in.t.shape
    dev = feats_in.t.device
    catbuf = Act(raw._new((n, h, w, 2 * mid), dtype=BF16, device=dev))     # [context | feats]
    feats = E.conv_bn(feats_in, p + ".conv3x3_ocr.0", p + ".conv3x3_ocr.1.0", 3, relu=True, bias=True,
                      out=catbuf.t[..., mid:])
    a = E.conv_bn(feats_in, p + ".aux_head.0", p + ".aux_head.1.0", 1, relu=True, bias=True)
    aux = E.conv_head(a, p + ".aux_head.2", bias=True)
    proxy = spatial_gather(E, feats, aux, K)
    ob = p + ".ocr_distri_head.object_context_block"
    q = E.conv_bn(feats, ob + ".f_pixel.0", ob + ".f_pixel.1.0", 1)
    q = E.conv_bn(q, ob + ".f_pixel.2", ob + ".f_pixel.3.0", 1)
    kk = E.conv_bn(proxy, ob + ".f_object.0", ob + ".f_object.1.0", 1)
    kk = E.conv_bn(kk, ob + ".f_object.2", ob + ".f_object.3.0", 1)
    vv = E.conv_bn(proxy, ob + ".f_down.0", ob + ".f_down.1.0", 1)
    ctx = object_attention(E, q, kk, vv, K)
    up = E.conv_bn(ctx, ob + ".f_up.0", ob + ".f_up.1.0", 1, out=catbuf.t[..., :mid])
    E.slice_marker(catbuf, [(up, 0, mid), (feats, mid, 2 * mid)])
    cb = p + ".ocr_distri_head.conv_bn_dropout"
    ocr_feats = E.conv_bn(catbuf, cb + ".0", cb + ".1.0", 1, relu=True,
                          post_scale=E.drop_mask if E.training else None)
    cls = E.conv_head(ocr_feats, p + ".cls_head", bias=True)
    return cls, aux, ocr_feats


def attn_head(E, x, ocfg=A.OCR_DEFAULT, drop_pass=0):
    """make_attn_head / old_make_attn_head (network/utils.py:343-382) in the variant ocfg selects (A.attn_head_plan):
    returns the PRE-sigmoid logit HeadRec ([N,h,w,1] fp32); the sigmoid is applied where the map is consumed (mscale
    kernels). In training, nn.Dropout(0.5) is fused into the last BatchNorm apply pass (and its backward) with keep bits
    drawn from E.attn_seed; drop_pass gives each scale pass of the step its own bits."""
    stages, last, drop = A.attn_head_plan(ocfg)
    t = x
    for i, (c, b) in enumerate(stages):
        d = (E.attn_seed, drop_pass) if drop and E.training and i == len(stages) - 1 else None
        t = E.conv_bn(t, c, b, 3, dropout=d)
    return E.conv_head(t, last, bias=False, ld=1)


def seg_head(E, x, p="seg_head"):
    """make_seg_head (network/utils.py:320-329) for basic.HRNet."""
    t = E.conv_bn(x, p + ".0", p + ".1", 3)
    t = E.conv_bn(t, p + ".3", p + ".4", 3)
    return E.conv_head(t, p + ".6", bias=False)


# ----------------------------------------------------------------------------------------------- DeepLabV3+ / WRN-38 (f2)
def wrn_block(E, p, x, in_ch, ch, stride, dil, drop_mask):
    """IdentityResidualBlock.forward (network/wider_resnet.py:170-183). x: raw (pre-activation) Act carrying its batch
    statistics; returns the raw residual sum (+ statistics from the last convolution's epilogue)."""
    a = E.preact(x, p + ".bn1.0")
    need_proj = stride != 1 or in_ch != ch[-1]
    short = E.conv_sum(a, p + ".proj_conv", 1, stride) if need_proj else x
    c = p + ".convs"
    if len(ch) == 2:
        t = E.conv_bn(a, c + ".conv1", c + ".bn2.0", 3, stride=stride, dilation=dil)
        return E.conv_sum(t, c + ".conv2", 3, 1, dil, addend=short, want_stats=True)
    t = E.conv_bn(a, c + ".conv1", c + ".bn2.0", 1, stride=stride)
    t = E.conv_bn(t, c + ".conv2", c + ".bn3.0", 3, dilation=dil, post_scale=drop_mask)
    return E.conv_sum(t, c + ".conv3", 1, 1, 1, addend=short, want_stats=True)


def aspp(E, x, red):
    """AtrousSpatialPyramidPoolingModule.forward (network/utils.py:207-218) at output stride 8 (rates 12 / 24 / 36):
    image pooling, the 1x1 and the three dilated 3x3 branches, each `red` channels wide, written into their slices of
    one concat Act [n, h, w, 5 * red] = [img | 1x1 | d12 | d24 | d36]."""
    n, h, w, _ = x.t.shape
    cat = Act(raw._new((n, h, w, 5 * red), dtype=BF16, device=x.t.device))
    img = E.conv_bn(E.image_pool(x), "aspp.img_conv.0", "aspp.img_conv.1", 1)
    pieces = [(E.broadcast(img, h, w, cat.t[..., 0:red]), 0, red)]
    one = E.conv_bn(x, "aspp.features.0.0", "aspp.features.0.1", 1, out=cat.t[..., red:2 * red])
    pieces.append((one, red, 2 * red))
    for i, r in enumerate(A.ASPP_RATES):
        c0 = (2 + i) * red
        f = "aspp.features.%d" % (i + 1)
        pieces.append((E.conv_bn(x, f + ".0", f + ".1", 3, dilation=r, out=cat.t[..., c0:c0 + red]), c0, c0 + red))
    E.slice_marker(cat, pieces)
    return cat


def deepv3_pass(E, images, wcfg, size_hw, drop_mask):
    """DeepV3Plus.forward up to the half-resolution logits (network/deepv3.py:75-88), MscaleV3Plus._fwd up to its two
    heads (network/mscale.py:296-316): WRN-38 trunk (output stride 8), ASPP (network/utils.py:204-216), decoder.
    size_hw: pass input size (ResizeX folded into image_prep); drop_mask: fp32 Dropout2d multipliers of mod6 / mod7
    in A.wrn_drop_layout order, or None. Returns (logit HeadRec [n, h/2, w/2, 19], decoder concat Act
    [n, h/2, w/2, 304] = [bot_fine(s2) | up(bot_aspp(aspp))])."""
    n = images.shape[0]
    x16 = Act(raw.image_prep(images, size_hw[0], size_hw[1]), needs_grad=False)
    x = E.conv_sum(x16, "backbone.mod1.conv1", 3)
    feats = {}
    drop_masks = {}
    if drop_mask is not None:
        off = 0
        for bp, c, _p in A.wrn_drop_layout(wcfg):
            drop_masks[bp] = drop_mask[off:off + n * c].view(n, c)
            off += n * c
    for mod, blk, in_ch, ch, stride, dil, drop in A.wrn_block_plan(wcfg):
        if blk == "block1" and mod in ("mod2", "mod3"):
            x = E.maxpool(x)                                               # pool2 / pool3
        bp = "backbone.%s.%s" % (mod, blk)
        dm = drop_masks.get(bp)
        x = wrn_block(E, bp, x, in_ch, ch, stride, dil, dm)
        feats[mod] = x
    s2, final = feats["mod2"], x
    dev = final.t.device
    conv_aspp = E.conv_sum(aspp(E, final, 256), "bot_aspp", 1)
    h2, w2 = s2.t.shape[1:3]
    cat2 = Act(raw._new((n, h2, w2, 48 + 256), dtype=BF16, device=dev))
    conv_s2 = E.conv_sum(s2, "bot_fine", 1, out=cat2.t[..., :48])
    up = E.fuse((n, h2, w2, 256), [("id", conv_aspp)], relu=False, out=cat2.t[..., 48:])
    E.slice_marker(cat2, [(conv_s2, 0, 48), (up, 48, 304)])
    t = E.conv_bn(cat2, "final.0", "final.1", 3)
    t = E.conv_bn(t, "final.3", "final.4", 3)
    return E.conv_head(t, "final.6", bias=False), cat2


# ----------------------------------------------------------------------------------------------- per-scale pass
def scale_pass(E, images, size_hw, arch, hcfg, ocfg, drop_mask=None, drop_pass=0):
    """MscaleOCR._fwd (network/ocrnet.py:170-183) up to the quarter-resolution maps (the x4 Upsample is fused into the
    blend/loss kernels). images: fp32 NCHW; size_hw: pass input size (ResizeX folded into image_prep).
    mscale.DeepV3W38: MscaleV3Plus._fwd (network/mscale.py:296-328) up to the half-resolution maps; drop_mask: this
    pass' WRN-38 Dropout2d multipliers (deepv3_pass). basic.HRNet_ASP / mscale.HRNet_ASP: the ASPP models over the
    HRNet trunk, up to their quarter-resolution maps. drop_pass: this pass' index in the attention head's dropout key
    (attn_head)."""
    if arch == "mscale.DeepV3W38":     # both heads read the decoder concat
        cls, cat = deepv3_pass(E, images, hcfg, size_hw, drop_mask)
        return dict(cls=cls, aux=None, attn=attn_head(E, cat, ocfg, drop_pass))
    x16 = Act(raw.image_prep(images, size_hw[0], size_hw[1]), needs_grad=False)
    feats = hrnet_forward(E, x16, hcfg)
    if A.has_hrnet_aspp(arch):
        # basic.ASPP.forward / mscale.ASPP._fwd (network/basic.py:84-92, network/mscale.py:496-511): ASPP on the
        # stride-4 trunk features, bot_aspp (1x1, no BN / ReLU), then the seg head and, for the mscale model, the
        # attention head on the same 256-channel map
        x = E.conv_sum(aspp(E, feats, ocfg["aspp_bot_ch"]), "bot_aspp", 1)
        cls = seg_head(E, x, "final")
        return dict(cls=cls, aux=None, attn=attn_head(E, x, ocfg, drop_pass) if arch == "mscale.HRNet_ASP" else None)
    if arch == "basic.HRNet":
        return dict(cls=seg_head(E, feats), aux=None, attn=None)
    if arch == "mscale.HRNet":      # MscaleBasic._fwd (network/mscale.py:463-470): both heads read the trunk features
        return dict(cls=seg_head(E, feats, "cls_head"), aux=None, attn=attn_head(E, feats, ocfg, drop_pass))
    cls, aux, mid_feats = ocr_block(E, feats, ocfg)
    attn = attn_head(E, mid_feats, ocfg, drop_pass) if arch == "ocrnet.HRNet_Mscale" else None
    return dict(cls=cls, aux=aux, attn=attn)


def train_loss(E, images, gts, arch, hcfg, ocfg, lo_scale=0.5, ocr_alpha=0.4, sup_wt=0.0, ignore_index=255, E_lo=None,
               loss_kind="ce", img_wt=(1.0, False), ocr_aux_rmi=False):
    """Training forward + loss. ocrnet.HRNet_Mscale: MscaleOCR.two_scale_forward (network/ocrnet.py:264-319);
    mscale.HRNet, mscale.DeepV3W38, mscale.HRNet_ASP: MscaleBase.two_scale_forward (network/mscale.py:182-220; one
    head, no auxiliary loss; the DeepLab model's maps are on the half-resolution grid of each pass);
    deepv3.DeepV3PlusW38: DeepV3Plus.forward (network/deepv3.py:73-96);
    ocrnet.HRNet: OCRNet.forward (:104-122); basic.HRNet: Basic.forward (network/basic.py:50-64); basic.HRNet_ASP:
    ASPP.forward (network/basic.py:84-101).
    Returns the fp32 loss vector [total, cls, aux, sup_lo, sup_hi, rmi, aux rmi, 0]; pushes the loss backward on the
    tape. loss_kind "ce": CrossEntropyLoss2d (loss/utils.py:133-134); "rmi": RMILoss (loss/rmi.py:70-215) = sigmoid BCE
    on every head (the auxiliary / supervised terms are called with do_rmi=False, network/ocrnet.py:303-318) plus the
    region-mutual-information term on the main prediction; ocr_aux_rmi (cfg.LOSS.OCR_AUX_RMI) calls the auxiliary head
    with do_rmi=True as well. "img_wt": ImageBasedCrossEntropyLoss2d (loss/utils.py:70-118) with
    img_wt = (upper_bound, round the weights through binary16), on every head and supervised term.

    E_lo (optional, two-scale only): a second engine with its own stream, gradient buffer and BN batch-statistics
    slots. The 0.5x and 1.0x passes are independent until the blend, so the low-resolution program is enqueued on
    E_lo.stream (a parallel branch of the captured CUDA graph) in forward and in backward; its small kernels fill the
    SMs the full-resolution pass leaves idle."""
    n, _, H, W = images.shape
    two_scale = A.is_two_scale(arch)
    lo = None
    main = torch.cuda.current_stream() if images.is_cuda else None
    par = two_scale and E_lo is not None and E_lo.stream is not None
    if not par:
        E_lo = E
    # WRN-38 Dropout2d multipliers: one set per scale pass, [lo | hi] when two-scale (each pass draws its own masks)
    lo_mask = hi_mask = None
    if A.has_wrn38_trunk(arch) and E.drop_mask is not None:
        hi_mask = E.drop_mask
        if two_scale:
            half = E.drop_mask.numel() // 2
            lo_mask, hi_mask = E.drop_mask[:half], E.drop_mask[half:]
    if two_scale:
        hm, wm = int(H * lo_scale), int(W * lo_scale)      # ResizeX: floor(in * scale)
        if par:
            E_lo.stream.wait_stream(main)
            with torch.cuda.stream(E_lo.stream):
                lo = scale_pass(E_lo, images, (hm, wm), arch, hcfg, ocfg, lo_mask, drop_pass=0)
        else:
            lo = scale_pass(E, images, (hm, wm), arch, hcfg, ocfg, lo_mask, drop_pass=0)
    if A.has_wrn38_trunk(arch) and not two_scale:
        hi = dict(cls=deepv3_pass(E, images, hcfg, (H, W), hi_mask)[0], aux=None, attn=None)
    else:
        hi = scale_pass(E, images, (H, W), arch, hcfg, ocfg, hi_mask, drop_pass=1)
    if par:
        main.wait_stream(E_lo.stream)
    nheads = 2 if A.has_ocr(arch) else 1
    hq, wq = hi["cls"].logits.shape[1:3]
    rmi = loss_kind == "rmi"
    kind = 1 if rmi else 0
    if two_scale:
        hl, wl = lo["cls"].logits.shape[1:3]
        d = raw.mscale_desc(n, H, W, hq, wq, hm, wm, hl, wl, nheads, 1.0, ocr_alpha, sup_wt, ignore_index, kind)
        lo_attn = lo["attn"].logits
        mid, mid_sup = raw.mscale_mid_fwd(d, lo["cls"].logits, lo["aux"].logits if nheads > 1 else None, lo_attn)
    else:
        d = raw.mscale_desc(n, H, W, hq, wq, 0, 0, 0, 0, nheads, 1.0, ocr_alpha, 0.0, ignore_index, kind)
        mid = mid_sup = None
    coef = None
    if loss_kind == "img_wt":
        # one histogram of the whole local batch per step; every head reads the same per-image coefficients
        _, _, coef, inv_count = raw.label_class_weights(gts, img_wt[0], img_wt[1])
    else:
        inv_count = raw.count_valid(gts, ignore_index, plus_one=rmi)
    dpr = terms = dpr_aux = terms_aux = None
    if rmi:
        pr, la = raw.rmi_pool(d, gts, hi["cls"].logits, mid)
        dpr, terms = raw.rmi_solve_grad(d, pr, la, d.w_head0)
        if ocr_aux_rmi and nheads > 1:
            pr_aux = raw.rmi_pool_aux(d, gts, hi["aux"].logits, mid)
            dpr_aux, terms_aux = raw.rmi_solve_grad(d, pr_aux, la, d.w_head1)
    loss, g_hi, g_lo, g_sup = raw.mscale_loss_fwd(d, gts, inv_count, hi["cls"].logits,
                                                  hi["aux"].logits if nheads > 1 else None, mid, mid_sup, dpr, terms,
                                                  coef, dpr_aux, terms_aux)

    def loss_bwd():
        d_cls, d_aux = raw.mscale_hi_bwd(d, g_hi)
        hi["cls"].dlogits = d_cls
        if nheads > 1:
            hi["aux"].dlogits = d_aux
        if two_scale:
            dl_cls, dl_aux, dl_attn = raw.mscale_lo_bwd(d, g_lo, g_sup, lo["cls"].logits,
                                                        lo["aux"].logits if nheads > 1 else None, lo_attn, mid)
            lo["cls"].dlogits, lo["attn"].dlogits = dl_cls, dl_attn
            if nheads > 1:
                lo["aux"].dlogits = dl_aux
            if par:
                # allocated on the main stream, consumed on the low-resolution stream: keep them until the final join
                E.hold.extend((dl_cls, dl_aux, dl_attn))
                E_lo.stream.wait_stream(main)
                with torch.cuda.stream(E_lo.stream):
                    E_lo.run_backward()        # whole 0.5x backward, concurrent with the 1.0x tape below
    E._push(loss_bwd)
    return loss


def run_backward(E, E_lo=None):
    """Backward of a step built by train_loss: E's tape on the current stream (its first entry forks E_lo's tape onto
    E_lo.stream), then the join."""
    E.run_backward()
    if E_lo is not None and E_lo.stream is not None:
        torch.cuda.current_stream().wait_stream(E_lo.stream)
        E_lo.finish()
    E.finish()
