"""fp32 restatement of the attention-head ablations of the multi-scale models (--mscale_no3x3, --mscale_dropout,
--mscale_old_arch; make_attn_head / old_make_attn_head / init_attn, network/utils.py:332-382) on the four archs that
build the head: ocrnet.HRNet_Mscale, mscale.HRNet, mscale.HRNet_ASP and mscale.DeepV3W38. The archs' oracles in
oracle/seg_oracle.py, tests/_hrnet_asp_oracle.py and tests/_mscale_deepv3_oracle.py call seg_oracle.attn_head by
attribute, so `head_variant` swaps in the variant's head for the duration of a run and leaves those files unchanged.
Pinned to the unmodified reference by tests/golden/reference_attn_head.pt (tests/golden/make_golden_attn_head.py).
Test infrastructure only."""
import contextlib

import torch
import torch.nn.functional as F

from oracle import seg_oracle as O

ARCHS = ("ocrnet.HRNet_Mscale", "mscale.HRNet", "mscale.HRNet_ASP", "mscale.DeepV3W38")
# name -> (MSCALE_INNER_3x3, MSCALE_DROPOUT, MSCALE_OLDARCH) (config.py:133-135)
VARIANTS = {
    "default": (True, False, False),
    "no3x3": (False, False, False),
    "dropout": (True, True, False),
    "oldarch": (True, False, True),
    "no3x3_dropout": (False, True, False),
}


def supported(arch, variant):
    """mscale.DeepV3W38 takes --mscale_no3x3 only; the model refuses the other two there. (It builds its trunk before
    the head, and WiderResNetA2.__init__ rebinds torch.nn.Dropout to Dropout2d, network/wider_resnet.py:302, so its
    `drop` would be a channel dropout.)"""
    return not (arch == "mscale.DeepV3W38" and (VARIANTS[variant][1] or VARIANTS[variant][2]))


def ocfg_keys(variant):
    inner, drop, old = VARIANTS[variant]
    return dict(mscale_inner_3x3=inner, mscale_dropout=drop, mscale_oldarch=old)


def head_layers(variant, p="scale_attn"):
    """-> ([(conv, bn) of each 3x3 + BN + ReLU stage], final 1x1 conv, has dropout). old_make_attn_head ignores the
    other two flags; make_attn_head names its layers conv0 / bn0 / [conv1 / bn1] / [drop] / conv2."""
    inner, drop, old = VARIANTS[variant]
    if old:
        return [(p + ".0", p + ".1"), (p + ".3", p + ".4")], p + ".6", False
    stages = [(p + ".conv0", p + ".bn0")] + ([(p + ".conv1", p + ".bn1")] if inner else [])
    return stages, p + ".conv2", drop


_DEFAULT_TO_OLD = {".conv0.": ".0.", ".bn0.": ".1.", ".conv1.": ".3.", ".bn1.": ".4.", ".conv2.": ".6."}


def rename_state_dict(sd, variant):
    """A synthetic state dict of the default head -> the variant's: the inner stage is dropped under no3x3, the old
    head renames its layers to nn.Sequential indices. Tensors keep their values (the scale_attn keys come last)."""
    inner, _drop, old = VARIANTS[variant]
    out = {}
    for k, v in sd.items():
        if k.startswith("scale_attn."):
            if old:
                for a, b in _DEFAULT_TO_OLD.items():
                    if k.startswith("scale_attn" + a):
                        k = "scale_attn" + b + k[len("scale_attn" + a):]
                        break
            elif not inner and (k.startswith("scale_attn.conv1.") or k.startswith("scale_attn.bn1.")):
                continue
        out[k] = v
    return out


def init_attn_(sd):
    """init_attn (network/utils.py:332-341) on the old head: every conv weight zero, BN (1, 0)."""
    for k, v in sd.items():
        if k.startswith("scale_attn.") and v.dim() == 4:
            v.zero_()
    return sd


def seeded_masks(seed):
    """Keep masks of nn.Dropout(0.5) regenerated from a seed: call k gets rand(shape, Generator(seed + k)) < 0.5. The
    golden script runs the reference with exactly these masks (lo pass first, then the 1.0x pass)."""
    calls = [0]

    def fn(shape):
        g = torch.Generator().manual_seed(seed + calls[0])
        calls[0] += 1
        return (torch.rand(tuple(shape), generator=g) < 0.5).float()
    return fn


def attn_head(ctx, p, x, variant, keep_fn=None):
    """The variant's head: stages of 3x3 conv + BN + ReLU, nn.Dropout(0.5) (training only; keep_fn(shape) -> 0/1
    NCHW mask, None = identity), 1x1 conv, sigmoid."""
    q = ctx.q
    stages, last, drop = head_layers(variant, p)
    for c, b in stages:
        x = q(F.relu(O.bn(ctx, b, q(O.conv(ctx, c, x, 1, 1)))))
    if drop and ctx.training and keep_fn is not None:
        x = x * keep_fn(x.shape).to(x.device) * 2.0
    return torch.sigmoid(ctx.qg(O.conv(ctx, last, x)))


@contextlib.contextmanager
def head_variant(variant, keep_fn=None):
    """Run seg_oracle-based models with the variant's attention head."""
    orig = O.attn_head
    O.attn_head = lambda ctx, p, x: attn_head(ctx, p, x, variant, keep_fn)
    try:
        yield
    finally:
        O.attn_head = orig


# ----------------------------------------------------------------------------------------------- per-arch plumbing
def _wcfg(hcfg):
    """mscale.DeepV3W38 takes its WRN-38 widths through `hcfg` (default: the reference's full widths)."""
    return hcfg if "structure" in hcfg else O.WRN38


def synth_state_dict(arch, variant, hcfg=O.HRNET_W16_TEST, seed=4):
    import _hrnet_asp_oracle as HA
    import _mscale_deepv3_oracle as MD
    if arch == "mscale.DeepV3W38":
        sd = MD.synth_state_dict(_wcfg(hcfg), seed=seed)
    elif arch == "mscale.HRNet_ASP":
        sd = HA.synth_state_dict(arch, hcfg, seed=seed)
    else:
        sd = O.synth_state_dict(arch, hcfg, seed=seed)
    return rename_state_dict(sd, variant)


def two_scale(arch, ctx, images, gts, criterion=O.criterion_ce, hcfg=O.HRNET_W16_TEST, sup_wt=0.0):
    import _hrnet_asp_oracle as HA
    import _mscale_deepv3_oracle as MD
    if arch == "ocrnet.HRNet_Mscale":
        ocfg = dict(O.OCR_CFG, dropout=0.0)
        return O.mscale_two_scale(ctx, images, gts, criterion, hcfg, ocfg, supervised_mscale_wt=sup_wt)
    if arch == "mscale.HRNet":
        return O.mscale_basic_two_scale(ctx, images, gts, criterion, hcfg, supervised_mscale_wt=sup_wt)
    if arch == "mscale.HRNet_ASP":
        return HA.two_scale(ctx, images, gts, criterion, hcfg, supervised_mscale_wt=sup_wt)
    return MD.two_scale(ctx, images, gts, criterion, _wcfg(hcfg), supervised_mscale_wt=sup_wt)


def nscale(arch, ctx, images, scales, hcfg=O.HRNET_W16_TEST):
    import _hrnet_asp_oracle as HA
    import _mscale_deepv3_oracle as MD
    if arch == "ocrnet.HRNet_Mscale":
        return O.mscale_nscale(ctx, images, scales, hcfg, dict(O.OCR_CFG, dropout=0.0))
    if arch == "mscale.HRNet":
        return O.mscale_basic_nscale(ctx, images, scales, hcfg)
    if arch == "mscale.HRNet_ASP":
        return HA.nscale(ctx, images, scales, hcfg)
    return MD.nscale(ctx, images, scales, _wcfg(hcfg))


def forward(arch, variant, ctx, images, gts=None, keep_fn=None, criterion=O.criterion_ce, hcfg=O.HRNET_W16_TEST,
            sup_wt=0.0, scales=None):
    """Training loss (two-scale) or evaluation outputs (two-scale, or n-scale with `scales`) of arch + variant."""
    with head_variant(variant, keep_fn):
        if ctx.training or scales is None:
            return two_scale(arch, ctx, images, gts, criterion, hcfg, sup_wt)
        return nscale(arch, ctx, images, scales, hcfg)


def oracle_train_step(arch, variant, hcfg, sd0, images, gts, keep_fn=None, sup_wt=0.0, crit=None, emulate_bf16=True,
                      device="cuda"):
    """tests/_parity.py oracle_train_step for arch + variant: -> (sd with .grad and updated running statistics, loss)."""
    import _parity as P
    P._tf32_off()
    sd = {k: v.clone().to(device) for k, v in sd0.items()}
    for k, v in sd.items():
        if v.is_floating_point() and "running" not in k:
            v.requires_grad_(True)
    ctx = O.Ctx(sd, training=True, emulate_bf16=emulate_bf16)
    loss = forward(arch, variant, ctx, images.to(device), gts.to(device), keep_fn, crit or O.criterion_ce, hcfg,
                   sup_wt)
    loss.backward()
    return sd, float(loss)


def noise_floor(arch, variant, hcfg, sd0, images, gts, sd_ref, keep_fn_factory=None, sup_wt=0.0, crit=None):
    """tests/_parity.py noise_floor for arch + variant (the same dropout masks on the one-ulp perturbed images)."""
    import _parity as P
    sd_p, _ = oracle_train_step(arch, variant, hcfg, sd0, P.ulp_perturbed(images), gts,
                                keep_fn_factory() if keep_fn_factory else None, sup_wt, crit)
    floor = {name: P.cos_rel(sd_p[name].grad, v.grad) for name, v in sd_ref.items()
             if v.grad is not None and float(v.grad.abs().max()) >= 1e-12}
    run = {k: float((sd_p[k] - v).abs().max() / (v.abs().max() + 1e-6)) for k, v in sd_ref.items()
           if k.endswith("running_mean") or k.endswith("running_var")}
    return floor, run
