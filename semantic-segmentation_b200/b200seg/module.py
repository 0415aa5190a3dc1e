"""``B200SegModule`` — the nn.Module the reference's ``network.get_model`` factory returns on the B200 path.

Contract mirrored from the reference (SURVEY.md §8b):
  * constructor ``f(num_classes, criterion)``; ``module(inputs)`` with ``inputs = {'images': fp32 [N,3,H,W],
    'gts': int64 [N,H,W]}``; train mode -> 0-dim loss tensor whose ``.backward()`` populates ``param.grad``; eval mode
    -> ``{'pred': [N,C,H,W], ...}`` (network/ocrnet.py:300-327, utils/trnval_utils.py:134-143);
  * ``state_dict()`` names / shapes / registration order identical to the reference module, parameters are ordinary
    fp32 ``nn.Parameter`` leaves (optimizers, DDP and checkpoints keep working); the bf16 operand layouts the kernels
    read are private caches refreshed from the master weights at the start of every step.

The training step executes forward AND backward inside ``forward()`` (the tape is static, so the whole step is one
CUDA graph after the first call); ``loss.backward()`` then only publishes the already-computed gradients into
``param.grad`` (accumulating if gradients are already present) and, under the DDP shim, all-reduces the flat buffer.
"""
import math

import torch
from torch import nn

from . import arch as A
from . import model as M
from . import raw
from .engine import BN_EPS, BN_MOMENTUM, Engine

F32 = torch.float32


def _criterion_kind(criterion):
    """Map the reference criterion object (loss/utils.py:40-67) to the fused loss implementation."""
    if criterion is None:
        return "ce"
    if isinstance(criterion, str):
        if criterion in ("ce", "rmi") or criterion.split(":")[0] == "img_wt":
            return criterion.split(":")[0]
        raise NotImplementedError("criterion %r: expected 'ce', 'rmi' or 'img_wt[:upper_bound[:half]]'" % criterion)
    name = type(criterion).__name__
    if name in ("CrossEntropyLoss2d", "CrossEntropyLoss"):
        return "ce"
    if name == "RMILoss":
        return "rmi"
    if name == "ImageBasedCrossEntropyLoss2d":
        return "img_wt"
    if name == "ImgWtLossSoftNLL":
        raise NotImplementedError(
            "criterion ImgWtLossSoftNLL (--jointwtborder) is not covered: it needs the multi-hot border targets of the "
            "dataset, and its forward(inputs, target) takes no do_rmi, so the reference itself raises a TypeError with "
            "these architectures")
    raise NotImplementedError("criterion %s is outside the B200 hot path (CE, RMI and image-weighted CE are covered)"
                              % name)


def _img_wt_options(criterion, ignore_index=255):
    """ImageBasedCrossEntropyLoss2d (loss/utils.py:70-118) -> (upper_bound, round the weights through binary16).
    The weights are rounded when cfg.BATCH_WEIGHTING is off and fp16 is on (weights.half(), read back as fp32 by
    apex's nll_loss). String form: 'img_wt[:upper_bound[:half]]'."""
    if isinstance(criterion, str):
        parts = criterion.split(":")
        return (float(parts[1]) if len(parts) > 1 else 1.0), (len(parts) > 2 and parts[2] == "half")
    if getattr(criterion, "norm", False):
        raise NotImplementedError("ImageBasedCrossEntropyLoss2d(norm=True) is not covered (get_loss never sets it)")
    if getattr(criterion, "num_classes", 19) != 19:
        raise NotImplementedError("ImageBasedCrossEntropyLoss2d: the class weights are instantiated for 19 classes")
    crit_ignore = getattr(getattr(criterion, "nll_loss", None), "ignore_index", ignore_index)
    if crit_ignore != ignore_index:
        raise NotImplementedError("ImageBasedCrossEntropyLoss2d: ignore_index %d differs from the model's %d"
                                  % (crit_ignore, ignore_index))
    return float(criterion.upper_bound), bool(criterion.fp16) and not bool(criterion.batch_weights)


def allreduce_sum_(flat):
    """Gradient all-reduce of the data-parallel step (collective C1, SURVEY.md §2b): ONE sum over the flat fp32 gradient
    buffer (NCCL over NVLink/NVSwitch on the GPU box, gloo in the CPU tests); returns the world size the caller divides
    by (folded into the publish kernel). No-op (returns 1) without a process group or with a single rank."""
    if not (torch.distributed.is_available() and torch.distributed.is_initialized()):
        return 1
    ws = torch.distributed.get_world_size()
    if ws > 1:
        torch.distributed.all_reduce(flat)
    return ws


def allreduce_mean_(flat):
    """all-reduce-average in place (host-logic helper of the CPU tests; the module folds the 1/world into its publish)."""
    ws = allreduce_sum_(flat)
    if ws > 1:
        flat.mul_(1.0 / ws)
    return flat


class _PublishGrads(torch.autograd.Function):
    """Bridges the engine's eagerly computed gradients into autograd: forward returns the loss, backward scales the
    step's gradient by the upstream gradient it receives and hands every parameter its slice of the flat buffer."""

    @staticmethod
    def forward(ctx, module, loss, anchor):
        ctx.module = module
        return loss.clone()

    @staticmethod
    def backward(ctx, grad_out):
        # grad_out is d(objective)/d(loss): 1 for loss.backward(), 1/k for (loss / k).backward() under gradient
        # accumulation, the loss scale under amp.scale_loss (train.py:499-505). Applied on the device (no host sync).
        ctx.module._publish(grad_out)
        return None, None, None


class B200SegModule(nn.Module):
    def __init__(self, arch, num_classes=19, criterion=None, hcfg=None, ocfg=None, lo_scale=0.5, ocr_alpha=0.4,
                 supervised_mscale_wt=0.0, ignore_index=255, n_scales=None, use_cuda_graph=True,
                 parallel_scales=True, syncbn=None, parallel_branches=True, ocr_aux_rmi=False, init_decoder=False):
        super().__init__()
        self.arch = arch
        self.criterion = criterion
        self.loss_kind = _criterion_kind(criterion)
        self.img_wt = _img_wt_options(criterion, ignore_index) if self.loss_kind == "img_wt" else (1.0, False)
        # cfg.LOSS.OCR_AUX_RMI: the auxiliary head is called with do_rmi=True (network/ocrnet.py:116,302-303); only the
        # RMILoss criterion reads do_rmi, and only the OCR architectures have an auxiliary head
        self.ocr_aux_rmi = bool(ocr_aux_rmi)
        self.is_deepv3 = A.has_wrn38_trunk(arch)
        # cfg.OPTIONS.INIT_DECODER (mscale.DeepV3W38): bot_fine, bot_aspp and scale_attn get initialize_weights too
        self.init_decoder = bool(init_decoder)
        self.hcfg = hcfg or (A.WRN38 if self.is_deepv3 else A.HRNET_W48)
        self._stem = "backbone.mod1.conv1.weight" if self.is_deepv3 else "backbone.conv1.weight"
        self.wrn_dropout_scale = 1.0     # tests set 0.0 for a dropout-free step
        self.ocfg = dict(A.OCR_DEFAULT, **(ocfg or {}))
        self.ocfg["num_classes"] = num_classes
        if num_classes != 19:
            raise NotImplementedError("the loss / soft-region kernels are instantiated for the 19 Cityscapes classes")
        red = self.ocfg["aspp_bot_ch"]
        if A.has_hrnet_aspp(arch) and (red <= 0 or red % 16):
            # bot_aspp reads the 5 * red channel concat: the weight-gradient GEMM takes input widths in whole
            # 16-channel groups (csrc/wgrad_igemm.cu)
            raise NotImplementedError("cfg.MODEL.ASPP_BOT_CH must be a positive multiple of 16 on the sm_90a "
                                      "convolutions; got %d" % red)
        if arch == "mscale.DeepV3W38" and self.ocfg["mscale_oldarch"]:
            raise NotImplementedError("cfg.MODEL.MSCALE_OLDARCH (--mscale_old_arch) is not provided on "
                                      "mscale.DeepV3W38: of the attention-head options only --mscale_no3x3 is")
        if arch == "mscale.DeepV3W38" and A.attn_head_plan(self.ocfg)[2]:
            # MscaleV3Plus builds the WRN-38 trunk first, and WiderResNetA2.__init__ rebinds torch.nn.Dropout to
            # Dropout2d for the whole process (network/wider_resnet.py:302): the head's `drop` is a channel dropout there
            raise NotImplementedError("cfg.MODEL.MSCALE_DROPOUT on mscale.DeepV3W38 is not covered: the reference's "
                                      "head dropout is Dropout2d(0.5) on that arch, only the element-wise "
                                      "Dropout(0.5) of the HRNet archs is on the sm_90a path")
        self.lo_scale, self.ocr_alpha, self.sup_wt, self.ignore_index = lo_scale, ocr_alpha, supervised_mscale_wt, ignore_index
        self.n_scales = n_scales
        self.use_cuda_graph = use_cuda_graph
        self.parallel_scales = parallel_scales     # run the 0.5x and 1.0x passes of the two-scale step concurrently
        self.parallel_branches = parallel_branches  # HRNet branches of a module on parallel streams
        # SyncBN (config.py:216-225, every scripts/*.yml sets syncbn: true): True = statistics of the global batch through
        # NVLink peer memory (needs torch.distributed, world > 1); None / False = per-GPU statistics. Opt-in for now: the
        # exchange was validated on 2 GPUs only.
        self.syncbn = syncbn
        self._sync = None
        self._run_flat = None
        self._specs = A.tensor_specs(arch, self.hcfg, self.ocfg)
        self._build_parameters()
        self._flat_grad = None
        self._packed = None
        self._planes = {}
        self._graphs = {}
        self._ddp_allreduce = False
        self._anchor = None

    # ------------------------------------------------------------------------------------------ parameters
    def _container(self, dotted):
        mod = self
        for part in dotted:
            if part not in mod._modules:
                mod.add_module(part, nn.Module())
            mod = mod._modules[part]
        return mod

    def _build_parameters(self):
        """Registers tensors under the reference names and reproduces its initialisation policy:
        backbone convs N(0, 1e-3), BN (1, 0) (network/hrnetv2.py:451-461); OCR / attention / seg heads keep the
        nn.Conv2d default (kaiming_uniform(a=sqrt(5)), bias U(+-1/sqrt(fan_in))) as in network/ocrnet.py:46-83.
        mscale.DeepV3W38 initialises only `final` (plus bot_* and scale_attn with init_decoder) with kaiming_normal_;
        ASPP and the rest keep the nn.Conv2d default (network/mscale.py:272-278). basic.HRNet_ASP initialises `final`,
        `bot_aspp` and `aspp` (network/basic.py:82), mscale.HRNet_ASP only `final` (network/mscale.py:494).
        The old attention head (cfg.MODEL.MSCALE_OLDARCH) is built by old_make_attn_head, whose init_attn zeroes its
        convolution weights (network/utils.py:332-341,381)."""
        if self.arch == "mscale.DeepV3W38":
            kaiming_normal = ("final", "bot_fine", "bot_aspp", "scale_attn") if self.init_decoder else ("final",)
        elif self.arch == "mscale.HRNet_ASP":
            kaiming_normal = ("final",)
        elif self.is_deepv3 or self.arch == "basic.HRNet_ASP":
            kaiming_normal = ("aspp", "bot_fine", "bot_aspp", "final")
        else:
            kaiming_normal = ()
        for name, shape, kind in self._specs:
            parts = name.split(".")
            owner = self._container(parts[:-1])
            leaf = parts[-1]
            in_backbone = parts[0] == "backbone"
            if kind == "conv_w":
                w = torch.empty(shape)
                if parts[0] in kaiming_normal:
                    # initialize_weights = kaiming_normal_ (network/deepv3.py:66-69, network/mynn.py:27-39)
                    nn.init.kaiming_normal_(w)
                elif parts[0] == "scale_attn" and self.ocfg["mscale_oldarch"]:
                    w.zero_()           # init_attn
                elif self.is_deepv3:
                    # WRN-38 trunk and the layers initialize_weights leaves alone: nn.Conv2d default
                    nn.init.kaiming_uniform_(w, a=math.sqrt(5))
                elif in_backbone:
                    nn.init.normal_(w, std=0.001)
                else:
                    nn.init.kaiming_uniform_(w, a=math.sqrt(5))
                owner.register_parameter(leaf, nn.Parameter(w))
            elif kind == "conv_b":
                wname = ".".join(parts[:-1]) + ".weight"
                fan_in = 1
                for nm, shp, _k in self._specs:
                    if nm == wname:
                        fan_in = shp[1] * shp[2] * shp[3]
                bound = 1.0 / math.sqrt(fan_in)
                owner.register_parameter(leaf, nn.Parameter(torch.empty(shape).uniform_(-bound, bound)))
            elif kind == "bn_w":
                owner.register_parameter(leaf, nn.Parameter(torch.ones(shape)))
            elif kind == "bn_b":
                owner.register_parameter(leaf, nn.Parameter(torch.zeros(shape)))
            elif kind == "bn_rm":
                owner.register_buffer(leaf, torch.zeros(shape))
            elif kind == "bn_rv":
                owner.register_buffer(leaf, torch.ones(shape))
            elif kind == "bn_nbt":
                owner.register_buffer(leaf, torch.tensor(0, dtype=torch.long))

    def _tensors(self):
        out = dict(self.named_parameters())
        out.update(dict(self.named_buffers()))
        return out

    def _ensure_device_state(self):
        """(Re)build the flat fp32 gradient buffer and the packed bf16 weight caches on the parameters' device."""
        params = [(n, p) for n, p in self.named_parameters()]
        dev = params[0][1].device
        if dev.type != "cuda":
            raise RuntimeError("B200SegModule runs on CUDA only (sm_90a); there is no CPU path - call .cuda() first")
        if self._flat_grad is None or self._flat_grad.device != dev:
            total = sum((p.numel() + 63) // 64 * 64 for _, p in params)
            self._flat_grad = torch.zeros(total, dtype=F32, device=dev)      # published gradients (param.grad views)
            self._step_flat = torch.zeros(total, dtype=F32, device=dev)      # gradient of the last executed step
            self._grad_views = {}
            off = 0
            for n, p in params:
                self._grad_views[n] = self._flat_grad[off:off + p.numel()].view(p.shape)
                off += (p.numel() + 63) // 64 * 64
            self._packed = {}
            # plane-ordered copies of the 3x3 operands that the halo-tile kernel streams its weights from (contiguous
            # bulk copies instead of 16-byte TMA rows), written by the same pack launch
            self._planes = {}
            for n, p in params:
                if p.dim() == 4:
                    o, i, k, _ = p.shape
                    if i == 3:      # stem: the image is padded to 16 channels (see resample_kernels.cu image_prep)
                        i = 16
                    w_f = torch.zeros((o, k * k, i), dtype=torch.bfloat16, device=dev)
                    w_d = torch.zeros((i, k * k, (o + 7) // 8 * 8), dtype=torch.bfloat16, device=dev)
                    self._packed[n[: -len(".weight")]] = (w_f, w_d)
                    imgs = tuple(raw.planes_image((o, i, k, k), which, dev) for which in (0, 1))
                    if imgs != (None, None):
                        self._planes[n[: -len(".weight")]] = imgs
            self._graphs = {}
            self._build_grad_accumulators(params, dev)
        self._ensure_flat_running(dev)

    def _build_grad_accumulators(self, params, dev):
        """Step-private fp32 gradient accumulators in the flat layout of ``_flat_grad`` (+ a tail for the stem, whose
        weight gradient accumulates on the 16-channel padded image):
          _acc_hi : everything the main (1.0x / only) pass produces - conv weights in the kernels' [O][taps][I] layout,
                    vectors (BN affine, biases) as is;
          _acc_lo : the same for the concurrently executed 0.5x pass.
        They are zeroed at the start of a step; ``raw.grad_fold`` sums and transposes them into ``_step_flat`` (OIHW) at
        its end. Nothing a step computes touches ``_flat_grad`` / ``param.grad`` before ``loss.backward()``."""
        total = self._flat_grad.numel()
        tail = 0
        for n, p in params:
            if p.dim() == 4 and p.shape[1] == 3:
                tail += p.shape[0] * p.shape[2] * p.shape[3] * 16
        self._acc_hi = torch.zeros(total + tail, dtype=F32, device=dev)
        self._acc_lo = torch.zeros(total + tail, dtype=F32, device=dev)
        self._eng_grads = {"hi": {}, "lo": {}}
        segs = []
        off, toff = 0, total
        for n, p in params:
            numel = p.numel()
            if p.dim() == 4:
                o, i, k, _ = p.shape
                if i == 3:
                    for which, acc in (("hi", self._acc_hi), ("lo", self._acc_lo)):
                        self._eng_grads[which][n] = acc[toff:toff + o * k * k * 16].view(o, k * k, 16)
                    segs.append((off, toff, o, i, k * k, 16))
                    toff += o * k * k * 16
                else:
                    for which, acc in (("hi", self._acc_hi), ("lo", self._acc_lo)):
                        self._eng_grads[which][n] = acc[off:off + numel].view(o, k * k, i)
                    segs.append((off, off, o, i, k * k, i))
            else:
                for which, acc in (("hi", self._acc_hi), ("lo", self._acc_lo)):
                    self._eng_grads[which][n] = acc[off:off + numel].view(p.shape)
                segs.append((off, off, 1, numel, 1, numel))
            off += (numel + 63) // 64 * 64
        self._fold_table = raw.grad_fold_table(segs, dev)

    def _engine_grads(self, which="hi"):
        """name -> fp32 tensor an Engine accumulates into."""
        return dict(self._eng_grads[which])

    def _fold_grads(self, with_lo):
        raw.grad_fold(self._step_flat, self._acc_hi, self._acc_lo if with_lo else None, self._fold_table, clear=False,
                      overwrite=True)

    def _ensure_flat_running(self, dev):
        """BatchNorm running statistics live in ONE flat fp32 buffer ([mean C | var C] per layer) and the module's
        registered buffers are views of it (state_dict / load_state_dict / checkpoints unchanged). That lets a step
        update every layer's running statistics with a single kernel after its concurrent scale passes have joined."""
        bn_names = [n[: -len(".running_mean")] for n, _s, k in self._specs if k == "bn_rm"]
        owners = [self._container(b.split(".")) for b in bn_names]
        ok = (self._run_flat is not None and self._run_flat.device == dev and
              all(o._buffers["running_mean"].device == dev for o in owners[:1]) and
              owners[0]._buffers["running_mean"].data_ptr() == self._run_flat.data_ptr() and
              owners[-1]._buffers["num_batches_tracked"].data_ptr() ==
              self._nbt_flat.data_ptr() + 8 * (len(owners) - 1))
        if ok:
            return
        total = sum(2 * o._buffers["running_mean"].numel() for o in owners)
        total = (total + 3) // 4 * 4
        flat = torch.zeros(total, dtype=F32, device=dev)
        nbt_flat = torch.zeros(len(owners), dtype=torch.long, device=dev)
        self._bn_slots = {}
        off = 0
        with torch.no_grad():
            for li, (b, o) in enumerate(zip(bn_names, owners)):
                c = o._buffers["running_mean"].numel()
                flat[off:off + c].copy_(o._buffers["running_mean"])
                flat[off + c:off + 2 * c].copy_(o._buffers["running_var"])
                nbt_flat[li].copy_(o._buffers["num_batches_tracked"])
                o._buffers["running_mean"] = flat[off:off + c]
                o._buffers["running_var"] = flat[off + c:off + 2 * c]
                o._buffers["num_batches_tracked"] = nbt_flat[li]
                self._bn_slots[b] = (off, c)
                off += 2 * c
        self._run_flat, self._nbt_flat = flat, nbt_flat
        # deferred BatchNorm finalisation (csrc/bn_fold.cuh): per pass and layer a forward cell pair
        # [2 * roundup16(c)] and a backward one [2 * c], one fp64 arena zeroed at the start of every step
        n_cells = sum(2 * ((c_ + 15) // 16 * 16) + 2 * c_ for _o, c_ in self._bn_slots.values())
        self._bncell_arena = torch.zeros(2 * n_cells, dtype=torch.float64, device=dev)
        self._bncells = []
        o = 0
        for _pass in range(2):
            cells = {}
            for b, (_o, c_) in self._bn_slots.items():
                cp = (c_ + 15) // 16 * 16
                cells[b] = (self._bncell_arena[o:o + 2 * cp], self._bncell_arena[o + 2 * cp:o + 2 * cp + 2 * c_])
                o += 2 * cp + 2 * c_
            self._bncells.append(cells)
        self._bstat = [torch.zeros(total, dtype=F32, device=dev) for _ in range(2)]
        self._bstat_views = [{b: t[o_:o_ + 2 * c_] for b, (o_, c_) in self._bn_slots.items()} for t in self._bstat]
        self._graphs = {}

    def _eval_bn_params(self):
        """Evaluation: scale / shift of EVERY BatchNorm layer from the running statistics in a handful of launches
        (instead of one per layer and pass): name -> (scale, shift) fp32 views."""
        dev = self._run_flat.device
        names = list(self._bn_slots)
        if getattr(self, "_eval_idx", None) is None or self._eval_idx[0].device != dev:
            im, iv, spans, o = [], [], {}, 0
            for b in names:
                off, c = self._bn_slots[b]
                im.append(torch.arange(off, off + c))
                iv.append(torch.arange(off + c, off + 2 * c))
                spans[b] = (o, o + c)
                o += c
            self._eval_idx = (torch.cat(im).to(dev), torch.cat(iv).to(dev), spans)
        im, iv, spans = self._eval_idx
        t = self._tensors()
        gamma = torch.cat([t[b + ".weight"].detach().reshape(-1) for b in names]).float()
        beta = torch.cat([t[b + ".bias"].detach().reshape(-1) for b in names]).float()
        scale = gamma * torch.rsqrt(self._run_flat[iv] + BN_EPS)
        shift = beta - self._run_flat[im] * scale
        return {b: (scale[a:z], shift[a:z]) for b, (a, z) in spans.items()}

    def _repack(self, side=None):
        """fp32 OIHW master weights -> bf16 kernel layouts, one launch for the whole model (inside the captured step:
        the weights change every optimizer step). With `side` (a stream) the data-gradient operands, which nothing
        reads before the backward, are packed there; returns the event the backward has to wait for."""
        convs = [(n, p) for n, p in self.named_parameters() if p.dim() == 4]
        ptrs = tuple(p.data_ptr() for _, p in convs)
        tab = getattr(self, "_pack_table", None)
        if tab is None or tab["ptrs"] != ptrs:
            entries = [(p.detach(), *self._packed[n[: -len(".weight")]],
                        *self._planes.get(n[: -len(".weight")], (None, None))) for n, p in convs]
            tab = self._pack_table = raw.pack_table(entries, convs[0][1].device)
            self._graphs = {}
        if side is None:
            raw.pack_weights(tab, 3)
            return None
        main = torch.cuda.current_stream()
        side.wait_stream(main)
        with torch.cuda.stream(side):
            raw.pack_weights(tab, 2)
            evt = torch.cuda.Event()
            evt.record()
        raw.pack_weights(tab, 1)
        return evt

    # ------------------------------------------------------------------------------------------ training step
    def _step_eager(self, images, gts, drop_mask, attn_seed=None):
        from . import _lib
        launches0 = _lib.KERNEL_LAUNCHES
        try:
            return self._step_body(images, gts, drop_mask, attn_seed)
        finally:
            raw.KEEP = None
            self.kernels_per_step = _lib.KERNEL_LAUNCHES - launches0   # same count when the captured graph replays

    def _sync_context(self):
        """Lazily builds the SyncBN mailboxes (collective: every rank must reach its first training step)."""
        if not self.syncbn:
            return None
        import torch.distributed as dist
        if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() < 2:
            return None
        if self._sync is None:
            from .p2p import SyncBNContext
            chans = {n[: -len(".running_mean")]: shp[0] for n, shp, k in self._specs if k == "bn_rm"}
            self._sync = SyncBNContext(chans, n_passes=2 if A.is_two_scale(self.arch) else 1)
            self._graphs = {}
        return self._sync

    def _step_body(self, images, gts, drop_mask, attn_seed=None):
        if getattr(self, "_side_stream", None) is None:
            self._side_stream = torch.cuda.Stream()
        sync = self._sync
        # SyncBN runs the same 21-stream program as per-GPU statistics: the one-warp waiter kernels never keep another
        # kernel from being scheduled (csrc/bn_kernels.cu), so up to eight exchanges (four branches x two passes) are in
        # flight and hide each other's NVLink round trips.
        wd_ready = self._repack(side=self._side_stream)
        if sync is not None:
            sync.advance()
        tensors = {k: v.detach() for k, v in self._tensors().items()}
        par = self.parallel_scales and A.is_two_scale(self.arch)
        # (one engine per scale pass, or a single pass: a layer's cells are used once per step)
        use_cells = sync is None and (par or not A.is_two_scale(self.arch))
        if use_cells:
            self._bncell_arena.zero_()
        self._acc_hi.zero_()         # two memsets (45 us each) beat clearing inside the fold's transposed gather
        if par:
            self._acc_lo.zero_()
        # every allocation of the step stays referenced until its final join (raw.py)
        raw.KEEP = []
        if getattr(self, "_bstreams", None) is None:
            mk = lambda: [torch.cuda.Stream() for _ in range(3)] if self.parallel_branches else []
            self._bstreams = {"hi": mk(), "lo": mk()}
            self._ws_holders = {"hi": [None], "lo": [None]}
        grads = self._engine_grads("hi")
        E_lo = None
        if par:
            if getattr(self, "_lo_stream", None) is None:
                self._lo_stream = torch.cuda.Stream()
                self._side_stream_lo = torch.cuda.Stream()
            grads_lo = self._engine_grads("lo")
            E_lo = Engine(tensors, grads_lo, self._packed, True, drop_mask, side_stream=self._side_stream_lo,
                          bstat=self._bstat_views[0], stream=self._lo_stream, sync=sync, pass_id=0,
                          branch_streams=self._bstreams["lo"], ws_holder=self._ws_holders["lo"],
                          bncells=self._bncells[0] if use_cells else None, attn_seed=attn_seed, planes=self._planes)
        two_pass = A.is_two_scale(self.arch)
        if sync is not None and two_pass and not par:
            raise RuntimeError("SyncBN needs parallel_scales=True for the two-scale step (one engine per pass)")
        E = Engine(tensors, grads, self._packed, True, drop_mask, side_stream=self._side_stream,
                   bstat=self._bstat_views[1] if par else None, sync=sync, pass_id=1 if two_pass else 0,
                   branch_streams=self._bstreams["hi"], ws_holder=self._ws_holders["hi"],
                   bncells=self._bncells[1] if use_cells else None, attn_seed=attn_seed, planes=self._planes)
        loss = M.train_loss(E, images, gts, self.arch, self.hcfg, self.ocfg, self.lo_scale, self.ocr_alpha, self.sup_wt,
                            self.ignore_index, E_lo=E_lo, loss_kind=self.loss_kind, img_wt=self.img_wt,
                            ocr_aux_rmi=self.ocr_aux_rmi)
        E.pre_backward_event = wd_ready
        if E_lo is not None:
            E_lo.pre_backward_event = wd_ready
        M.run_backward(E, E_lo)
        self._fold_grads(par)
        if par:
            assert E.bn_seen == E_lo.bn_seen and len(E.bn_seen) == len(self._bn_slots), "BN bookkeeping out of sync"
            raw.bn_running_update(self._run_flat, self._bstat[0], self._bstat[1], BN_MOMENTUM, self._nbt_flat, 2)
        raw.KEEP = None
        return loss

    def _drop_mask(self, n, device):
        """Dropout2d(0.05) channel mask (network/ocr_utils.py:146) drawn from torch's generator, folded with 1/(1-p)."""
        if self.is_deepv3:
            # WRN-38 mod6 / mod7: Dropout2d(0.3) / Dropout2d(0.5) in front of conv3 (network/wider_resnet.py:302 patches
            # nn.Dropout to Dropout2d; :336-338). One flat fp32 buffer, [n, c] per block in A.wrn_drop_layout order;
            # the two-scale step draws a set per pass, the 0.5x pass first (network/mscale.py:188-192): [lo | hi].
            parts = []
            for _pass in range(2 if A.is_two_scale(self.arch) else 1):
                for _bp, c, p in A.wrn_drop_layout(self.hcfg):
                    p = p * self.wrn_dropout_scale
                    keep = torch.bernoulli(torch.full((n * c,), 1.0 - p, dtype=F32, device=device))
                    parts.append(keep / (1.0 - p))
            return torch.cat(parts) if parts else None
        if not A.has_ocr(self.arch):
            return None
        p = self.ocfg["dropout"]
        c = self.ocfg["mid_channels"]
        if p == 0.0:
            return torch.ones((n, c), dtype=F32, device=device)
        keep = torch.bernoulli(torch.full((n, c), 1.0 - p, dtype=F32, device=device))
        return keep / (1.0 - p)

    def _attn_seed(self, device):
        """Key of the attention head's element-wise Dropout(0.5) (cfg.MODEL.MSCALE_DROPOUT) for one step: an int64 drawn
        on the device from torch's CUDA generator (no host synchronisation); the kernels derive every keep bit from it
        (csrc/dropout.cuh), so no mask is stored. None when the head has no dropout."""
        if not (A.is_two_scale(self.arch) and A.attn_head_plan(self.ocfg)[2]):
            return None
        return torch.randint(-2 ** 63, 2 ** 63 - 1, (1,), dtype=torch.int64, device=device)

    def _train_forward(self, images, gts):
        self._ensure_device_state()
        self._sync_context()
        images = images.contiguous().float()
        gts = gts.contiguous().long()
        key = (tuple(images.shape), str(images.device))
        mask = self._drop_mask(images.shape[0], images.device)
        seed = self._attn_seed(images.device)
        self.last_attn_seed = seed
        if not self.use_cuda_graph:
            return self._step_eager(images, gts, mask, seed)
        st = self._graphs.get(key)
        if st is None:
            st = dict(images=images.clone(), gts=gts.clone(), mask=None if mask is None else mask.clone(),
                      seed=None if seed is None else seed.clone(), calls=0, graph=None, loss=None)
            self._graphs[key] = st
        st["images"].copy_(images)
        st["gts"].copy_(gts)
        if mask is not None:
            st["mask"].copy_(mask)
        if seed is not None:
            st["seed"].copy_(seed)
        st["calls"] += 1
        if st["graph"] is None:
            if st["calls"] < 2:      # first call: eager warm-up (sets kernel attributes, fills the allocator pools)
                return self._step_eager(st["images"], st["gts"], st["mask"], st["seed"])
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                st["loss"] = self._step_eager(st["images"], st["gts"], st["mask"], st["seed"])
            st["graph"] = g
        st["graph"].replay()
        return st["loss"]

    def _publish(self, grad_out=None):
        """Called from loss.backward(): param.grad (+)= grad_out * (gradient of the last step), averaged across the
        data-parallel ranks (collective C1) under the DDP shim. Contract, like autograd's: gradients the caller dropped
        (``zero_grad(set_to_none=True)``) are replaced, live ones are accumulated into. Every ``param.grad`` this creates
        is a view of ONE flat fp32 buffer (what FusedSGD and the all-reduce work on)."""
        scale = 1.0
        if self._ddp_allreduce:
            scale = 1.0 / allreduce_sum_(self._step_flat)
        if grad_out is not None:
            grad_out = grad_out.detach().reshape(()).to(F32)
        params = list(self.named_parameters())
        views = self._grad_views
        n_none = sum(1 for _, p in params if p.grad is None)
        if n_none == len(params):
            raw.publish_grads(self._flat_grad, self._step_flat, grad_out, scale, accumulate=False)
            for n, p in params:
                p.grad = views[n]
            return
        if n_none == 0 and all(p.grad.data_ptr() == views[n].data_ptr() for n, p in params):
            raw.publish_grads(self._flat_grad, self._step_flat, grad_out, scale, accumulate=True)
            return
        # mixed / foreign .grad tensors (rare: a caller that assigns its own gradient tensors): per-parameter slow path
        tmp = torch.empty_like(self._step_flat)
        raw.publish_grads(tmp, self._step_flat, grad_out, scale, accumulate=False)
        off = 0
        for n, p in params:
            t = tmp[off:off + p.numel()].view(p.shape)
            if p.grad is None:
                views[n].copy_(t)
                p.grad = views[n]
            else:
                p.grad.add_(t)
            off += (p.numel() + 63) // 64 * 64

    # ------------------------------------------------------------------------------------------ forward
    def forward(self, inputs):
        assert "images" in inputs
        images = inputs["images"]
        if self.training:
            assert "gts" in inputs
            loss5 = self._train_forward(images, inputs["gts"])
            self.last_loss_terms = loss5
            if self._anchor is None or self._anchor.device != loss5.device:
                self._anchor = torch.zeros(1, device=loss5.device, requires_grad=True)
            return _PublishGrads.apply(self, loss5[0], self._anchor)
        return self._eval_forward(images)

    def _eval_forward(self, images):
        """Eval mode: the first call for an input shape runs eagerly, the second is captured into a CUDA graph (about a
        thousand launches per scale pass), later calls replay it. The returned maps are fresh tensors (copies of the
        graph's static outputs), so callers may keep them across calls like the reference's."""
        from .evalpath import eval_forward
        if not self.use_cuda_graph or not images.is_cuda:
            return eval_forward(self, images)
        self._ensure_device_state()
        images = images.contiguous().float()
        key = ("eval", tuple(images.shape), str(images.device), tuple(self.n_scales or ()))
        st = self._graphs.get(key)
        if st is None:
            st = dict(images=images.clone(), calls=0, graph=None, out=None)
            self._graphs[key] = st
        st["calls"] += 1
        if st["graph"] is None:
            if st["calls"] < 2:
                return eval_forward(self, images)
            st["images"].copy_(images)
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                st["out"] = eval_forward(self, st["images"])
            st["graph"] = g
        st["images"].copy_(images)
        st["graph"].replay()
        return {k: v.clone() for k, v in st["out"].items()}
