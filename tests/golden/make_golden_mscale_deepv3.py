"""Generates tests/golden/reference_mscale_deepv3.pt: outputs of the UNMODIFIED reference arch `mscale.DeepV3W38`
(MscaleV3Plus over the WideResNet-38 trunk, network/mscale.py:232-336) on CPU. Build container only:
    python tests/golden/make_golden_mscale_deepv3.py
Full-width WRN-38 (the reference hard-codes its widths) on 2 x 64 x 128 crops, dropout off, weights / inputs regenerated
by the tests from tests/_mscale_deepv3_oracle.synth_state_dict and oracle.seg_oracle.synth_batch. Also stores the
convolution FLOPs of the reference module's two scale passes at 1024 x 2048, counted with forward hooks on the meta
device, for the program-structure test."""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "semantic-segmentation_b200", "shims"))
sys.path.insert(1, "/root/reference")

import numpy as np
import torch

np.int = int
torch.cuda.DoubleTensor = torch.DoubleTensor
from oracle import seg_oracle as O  # noqa: E402
import _mscale_deepv3_oracle as MD  # noqa: E402
from config import cfg  # noqa: E402

torch.set_num_threads(8)
cfg.MODEL.BNFUNC = torch.nn.BatchNorm2d
cfg.MODEL.HRNET_CHECKPOINT = ""
cfg.DATASET.NUM_CLASSES = 19
cfg.DATASET.IGNORE_LABEL = 255
cfg.OPTIONS.TORCH_VERSION = 2.1

import network.wider_resnet as wr  # noqa: E402

_orig_init = wr.wrn38.__init__


def _init_no_ckpt(self, pretrained=True):          # the pretrained trunk file does not exist offline
    _orig_init(self, pretrained=False)


wr.wrn38.__init__ = _init_no_ckpt
import network.mscale as ref_mscale  # noqa: E402
from loss.utils import CrossEntropyLoss2d  # noqa: E402
from loss.rmi import RMILoss  # noqa: E402

GRADS = ("backbone.mod1.conv1.weight", "backbone.mod4.block2.convs.conv2.weight",
         "backbone.mod6.block1.convs.conv2.weight", "aspp.features.2.0.weight", "aspp.img_conv.0.weight",
         "bot_fine.weight", "bot_aspp.weight", "final.0.weight", "final.6.weight", "scale_attn.conv0.weight",
         "scale_attn.bn0.weight", "scale_attn.conv1.weight", "scale_attn.conv2.weight")


def _net(crit):
    net = ref_mscale.DeepV3W38(num_classes=19, criterion=crit)
    for m in net.modules():
        if isinstance(m, (torch.nn.Dropout2d, torch.nn.Dropout)):
            m.p = 0.0
    return net


def conv_flops(net, h, w, scale):
    """{conv module name: 2 * MACs} of one MscaleV3Plus._fwd at scale x (h, w) (meta tensors, eval mode)."""
    flops = {}
    hooks = []
    for name, m in net.named_modules():
        if isinstance(m, torch.nn.Conv2d):
            def hook(mod, inp, out, name=name):
                n, co, ho, wo = out.shape
                kh, kw = mod.kernel_size
                flops[name] = 2 * n * ho * wo * co * (mod.in_channels // mod.groups) * kh * kw
            hooks.append(m.register_forward_hook(hook))
    x = torch.empty((1, 3, h, w), device="meta")
    with torch.no_grad():
        net._fwd(x if scale == 1.0 else ref_mscale.ResizeX(x, scale))
    for hk in hooks:
        hk.remove()
    return flops


def main():
    out = {}
    sd = MD.synth_state_dict(O.WRN38, seed=4)
    images, gts = O.synth_batch(2, 64, 128, seed=6)
    for loss_name, sup in (("ce", 0.0), ("ce", 0.05), ("rmi", 0.05)):
        cfg.LOSS.SUPERVISED_MSCALE_WT = sup
        crit = CrossEntropyLoss2d(ignore_index=255) if loss_name == "ce" else RMILoss(num_classes=19, ignore_index=255)
        net = _net(crit)
        keys = list(net.state_dict().keys())
        assert keys == list(sd.keys()), [k for k in keys if k not in sd][:5] + [k for k in sd if k not in keys][:5]
        for k, v in net.state_dict().items():
            assert tuple(v.shape) == tuple(sd[k].shape), k
        net.load_state_dict(sd)
        net.train()
        loss = net({"images": images, "gts": gts})
        loss.backward()
        named = dict(net.named_parameters())
        after = net.state_dict()
        key = "%s/sup%g" % (loss_name, sup)
        out[key] = dict(loss=loss.detach().clone(), grads={n: O.sample_like(named[n].grad) for n in GRADS},
                        running_mean_attn_bn0=after["scale_attn.bn0.running_mean"].clone(),
                        running_var_attn_bn0=after["scale_attn.bn0.running_var"].clone(),
                        nbt_attn_bn0=int(after["scale_attn.bn0.num_batches_tracked"]),
                        running_var_mod5=after["backbone.mod5.block3.convs.bn2.0.running_var"].clone())
        print(key, float(loss))
        if key == "ce/sup0":
            net.eval()
            with torch.no_grad():
                cfg.MODEL.N_SCALES = None
                o2 = net({"images": images})
                cfg.MODEL.N_SCALES = [0.5, 1.0, 2.0]
                o3 = net({"images": images})
                cfg.MODEL.N_SCALES = None
            out["eval_two_scale"] = {k: O.sample_like(v) for k, v in o2.items()}
            out["eval_two_scale_keys"] = sorted(o2.keys())
            out["eval_three_scale"] = {k: O.sample_like(v) for k, v in o3.items()}
            out["eval_three_scale_keys"] = sorted(o3.keys())
            out["state_dict_keys"] = keys
            out["shapes"] = [tuple(v.shape) for v in net.state_dict().values()]
            out["param_order"] = [n for n, _ in net.named_parameters()]
            out["nparams"] = sum(p.numel() for p in net.parameters())
    cfg.LOSS.SUPERVISED_MSCALE_WT = 0.0
    net = _net(None).to("meta").eval()
    out["conv_flops_1024x2048"] = {"1.0": conv_flops(net, 1024, 2048, 1.0), "0.5": conv_flops(net, 1024, 2048, 0.5)}
    print("keys", len(out["state_dict_keys"]), "params", out["nparams"],
          "fwd TFLOP 1.0x %.4f 0.5x %.4f" % tuple(sum(v.values()) / 1e12 for v in out["conv_flops_1024x2048"].values()))
    torch.save(out, os.path.join(HERE, "reference_mscale_deepv3.pt"))
    print("wrote", os.path.getsize(os.path.join(HERE, "reference_mscale_deepv3.pt")), "bytes")


if __name__ == "__main__":
    main()
