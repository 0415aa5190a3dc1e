"""Shared constructor: reads the reference cfg keys the original modules read (SURVEY.md §5 'Config / flags')."""
import os
import sys

_PKG = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if _PKG not in sys.path:
    sys.path.insert(0, _PKG)

from b200seg import arch as A            # noqa: E402
from b200seg.module import B200SegModule  # noqa: E402


def build(arch, num_classes, criterion):
    kw = {}
    try:
        from config import cfg
        if not A.has_wrn38_trunk(arch):
            kw["hcfg"] = A.hrnet_cfg_from_reference_cfg(cfg)
        if arch == "mscale.DeepV3W38":
            kw["init_decoder"] = bool(getattr(getattr(cfg, "OPTIONS", None), "INIT_DECODER", False))
        ocfg = dict(A.OCR_DEFAULT)
        ocfg["mid_channels"] = cfg.MODEL.OCR.MID_CHANNELS
        ocfg["key_channels"] = cfg.MODEL.OCR.KEY_CHANNELS
        ocfg["segattn_bot_ch"] = cfg.MODEL.SEGATTN_BOT_CH
        if A.has_hrnet_aspp(arch):
            ocfg["aspp_bot_ch"] = int(cfg.MODEL.ASPP_BOT_CH)      # --aspp_bot_ch (config.py:131,313)
        kw["ocfg"] = ocfg
        kw["lo_scale"] = cfg.MODEL.MSCALE_LO_SCALE
        kw["ocr_alpha"] = cfg.LOSS.OCR_ALPHA
        kw["supervised_mscale_wt"] = cfg.LOSS.SUPERVISED_MSCALE_WT
        kw["ignore_index"] = cfg.DATASET.IGNORE_LABEL
        kw["n_scales"] = cfg.MODEL.N_SCALES
        if cfg.MODEL.ALIGN_CORNERS:
            raise NotImplementedError("align_corners=True is not covered by the B200 resampling kernels")
        if cfg.MODEL.OCR_ASPP:
            raise NotImplementedError("cfg.MODEL.OCR_ASPP (--ocr_aspp) is not covered: the reference itself raises "
                                      "NameError: name 'get_aspp' is not defined for it (network/ocr_utils.py never "
                                      "imports get_aspp)")
        # the attention-head ablations (--mscale_no3x3 / --mscale_dropout / --mscale_old_arch, config.py:318-325),
        # read by make_attn_head; archs without an attention head ignore them like the reference does
        ocfg["mscale_inner_3x3"] = bool(cfg.MODEL.MSCALE_INNER_3x3)
        ocfg["mscale_dropout"] = bool(cfg.MODEL.MSCALE_DROPOUT)
        ocfg["mscale_oldarch"] = bool(cfg.MODEL.MSCALE_OLDARCH)
        kw["ocr_aux_rmi"] = bool(cfg.LOSS.OCR_AUX_RMI)
        # cfg.MODEL.BNFUNC (config.py:216-225: apex.parallel.SyncBatchNorm under --syncbn --apex, else BatchNorm2d)
        # decides whether BatchNorm statistics span the data-parallel group
        bnfunc = getattr(cfg.MODEL, "BNFUNC", None)
        kw["syncbn"] = bnfunc is not None and "sync" in getattr(bnfunc, "__name__", str(bnfunc)).lower()
        # cfg.MODEL.HRNET_CHECKPOINT hangs off the hard-coded cfg.ASSETS_PATH (config.py:52,147) users edit in their
        # checkout; B200SEG_HRNET_CHECKPOINT overrides it without touching the reference ("" = random initialisation)
        checkpoint = os.environ.get("B200SEG_HRNET_CHECKPOINT", getattr(cfg.MODEL, "HRNET_CHECKPOINT", ""))
    except ImportError:
        checkpoint = ""
    if num_classes != 19:
        raise NotImplementedError("the B200 loss / soft-region kernels are instantiated for the 19 Cityscapes classes "
                                  "(csrc/mscale_common.cuh NC); got num_classes=%d" % num_classes)
    net = B200SegModule(arch, num_classes=num_classes, criterion=criterion, **kw)
    load_backbone_checkpoint(net, checkpoint)
    return net


def load_backbone_checkpoint(net, path):
    """HighResolutionNet.init_weights (network/hrnetv2.py:451-477): after the N(0, 1e-3) / (1, 0) initialisation the
    ImageNet-pretrained trunk is loaded into ``backbone.*`` with the reference's key remapping ('last_layer' ->
    'aux_head', 'model.' stripped; keys the trunk does not own are dropped); an empty path keeps the random init, a
    non-empty missing path raises like the reference does."""
    import torch
    if not path:
        return 0
    if not os.path.isfile(path):
        raise RuntimeError("No such file {}".format(path))
    pretrained = torch.load(path, map_location="cpu")
    own = net.state_dict()
    loaded = 0
    with torch.no_grad():
        for k, v in pretrained.items():
            k = "backbone." + k.replace("last_layer", "aux_head").replace("model.", "")
            if k in own and tuple(own[k].shape) == tuple(v.shape):
                own[k].copy_(v)
                loaded += 1
    return loaded
