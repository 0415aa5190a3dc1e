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
        if criterion in ("ce", "rmi"):
            return criterion
        raise NotImplementedError("criterion %r: expected 'ce' or 'rmi'" % criterion)
    name = type(criterion).__name__
    if name in ("CrossEntropyLoss2d", "CrossEntropyLoss"):
        return "ce"
    if name == "RMILoss":
        return "rmi"
    raise NotImplementedError("criterion %s is outside the B200 hot path (CE and RMI are covered)" % name)


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
                 parallel_scales=True, syncbn=None, parallel_branches=True):
        super().__init__()
        self.arch = arch
        self.criterion = criterion
        self.loss_kind = _criterion_kind(criterion)
        self.is_deepv3 = arch == "deepv3.DeepV3PlusW38"
        self.hcfg = hcfg or (A.WRN38 if self.is_deepv3 else A.HRNET_W48)
        self._stem = "backbone.mod1.conv1.weight" if self.is_deepv3 else "backbone.conv1.weight"
        self.wrn_dropout_scale = 1.0     # tests set 0.0 for a dropout-free step
        self.ocfg = dict(ocfg or A.OCR_DEFAULT)
        self.ocfg["num_classes"] = num_classes
        if num_classes != 19:
            raise NotImplementedError("the loss / soft-region kernels are instantiated for the 19 Cityscapes classes")
        self.lo_scale, self.ocr_alpha, self.sup_wt, self.ignore_index = lo_scale, ocr_alpha, supervised_mscale_wt, ignore_index
        self.n_scales = n_scales
        self.use_cuda_graph = use_cuda_graph
        self.parallel_scales = parallel_scales     # run the 0.5x and 1.0x passes of the two-scale step concurrently
        self.parallel_branches = parallel_branches  # HRNet branches of a module on parallel streams
        # SyncBN (config.py:216-225, every scripts/*.yml sets syncbn: true): True = statistics of the global batch through
        # NVLink peer memory (needs torch.distributed, world > 1); None / False = per-GPU statistics. Opt-in for now: the
        # exchange was validated on 2 GPUs only.
        self.syncbn = syncbn
        # BatchNorm statistics finalised inside the producing launches (csrc/bn_fold.cuh): 1262 launches fewer per step,
        # but measured 0.9 ms SLOWER on the device (40.18 vs 39.3 ms, alternating runs on one box: the tail of every
        # convolution grows by ~4 us while the removed finalisers ran on a handful of SMs next to other work) with no
        # clear end-to-end gain, so it is opt-in (B200SEG_FUSED_BN=1); SyncBN always uses the separate finaliser.
        import os
        self.fused_bn_finalize = os.environ.get("B200SEG_FUSED_BN", "0") == "1"
        # Deferred finalisation (default): the convolution / the backward reduction add their sums to per-layer fp64
        # cells and the consuming apply pass folds them in its prologue - no finaliser launch and no last-CTA tail on
        # the chain conv -> BN -> conv (B200SEG_BN_CELLS=0: separate bn_finalize / bn_bwd_finalize launches).
        self.bn_cells = os.environ.get("B200SEG_BN_CELLS", "1") == "1" and not self.fused_bn_finalize
        self._sync = None
        self._run_flat = None
        self._specs = A.tensor_specs(arch, self.hcfg, self.ocfg)
        self._build_parameters()
        self._flat_grad = None
        self._packed = None
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
        nn.Conv2d default (kaiming_uniform(a=sqrt(5)), bias U(+-1/sqrt(fan_in))) as in network/ocrnet.py:46-83."""
        for name, shape, kind in self._specs:
            parts = name.split(".")
            owner = self._container(parts[:-1])
            leaf = parts[-1]
            in_backbone = parts[0] == "backbone"
            if kind == "conv_w":
                w = torch.empty(shape)
                if self.is_deepv3:
                    # WRN-38 trunk: nn.Conv2d default; ASPP / bot_* / final: initialize_weights = kaiming_normal_
                    # (network/deepv3.py:66-69, network/mynn.py:27-39)
                    if in_backbone:
                        nn.init.kaiming_uniform_(w, a=math.sqrt(5))
                    else:
                        nn.init.kaiming_normal_(w)
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
            for n, p in params:
                if p.dim() == 4:
                    o, i, k, _ = p.shape
                    if i == 3:      # stem: the image is padded to 16 channels (see resample_kernels.cu image_prep)
                        i = 16
                    w_f = torch.zeros((o, k * k, i), dtype=torch.bfloat16, device=dev)
                    w_d = torch.zeros((i, k * k, (o + 7) // 8 * 8), dtype=torch.bfloat16, device=dev)
                    self._packed[n[: -len(".weight")]] = (w_f, w_d)
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
        # Gradient buckets for the overlapped data-parallel all-reduce, contiguous in the flat layout (= registration
        # order) and listed in the order the backward completes them: heads, transition3 + stage4, everything before.
        names = [n for n, _ in params]
        i1 = next((i for i, n in enumerate(names) if n.startswith("backbone.transition3.")), 0)
        i2 = next((i for i, n in enumerate(names) if not n.startswith("backbone.")), len(names))
        i1 = min(i1, i2)
        self._buckets = []
        for tag, (a, b) in (("heads", (i2, len(names))), ("stage4", (i1, i2)), ("rest", (0, i1))):
            if b > a:
                lo = segs[a][0]
                hi = segs[b - 1][0] + (segs[b - 1][2] * segs[b - 1][3] * segs[b - 1][4] + 63) // 64 * 64
                self._buckets.append(dict(tag=tag, lo=lo, hi=hi, table=raw.grad_fold_table(segs[a:b], dev)))

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
        # self-clearing reduction cells of the in-launch BatchNorm finalisation (raw.conv2d_fwd_bn), one set per pass
        self._bnfold = []
        for _pass in range(2):
            cells = {}
            acc = torch.zeros(sum(2 * ((c_ + 15) // 16 * 16) for _o, c_ in self._bn_slots.values()), dtype=torch.float64,
                              device=dev)
            tickets = torch.zeros(len(self._bn_slots), dtype=torch.int32, device=dev)
            o = 0
            for li, (b, (_o, c_)) in enumerate(self._bn_slots.items()):
                cp = (c_ + 15) // 16 * 16
                cells[b] = (acc[o:o + 2 * cp], tickets[li:li + 1])
                o += 2 * cp
            self._bnfold.append(cells)
        # deferred BatchNorm finalisation (csrc/bn_fold.cuh, counter == NULL): per pass and layer a forward cell pair
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
        (instead of one bn_eval_params launch per layer and pass): name -> (scale, shift) fp32 views."""
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
            entries = [(p.detach(), *self._packed[n[: -len(".weight")]]) for n, p in convs]
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
    def _step_eager(self, images, gts, drop_mask):
        from . import _lib
        launches0 = _lib.KERNEL_LAUNCHES
        try:
            if not self._prio():
                return self._step_body(images, gts, drop_mask)
            # B200SEG_PRIO=1 (experiment): the scale passes and their branch streams run on high-priority streams, the
            # weight-gradient / repack side streams (which feed nothing downstream inside the step) stay at the default
            # priority; kernel-node priorities are captured into the graph
            if getattr(self, "_prio_stream", None) is None:
                self._prio_stream = torch.cuda.Stream(priority=-1)
            cur = torch.cuda.current_stream()
            self._prio_stream.wait_stream(cur)
            with torch.cuda.stream(self._prio_stream):
                loss = self._step_body(images, gts, drop_mask)
            cur.wait_stream(self._prio_stream)
            loss.record_stream(cur)
            return loss
        finally:
            raw.KEEP = None
            self.kernels_per_step = _lib.KERNEL_LAUNCHES - launches0   # same count when the captured graph replays

    @staticmethod
    def _prio():
        import os
        return os.environ.get("B200SEG_PRIO", "0") == "1"

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

    def _step_body(self, images, gts, drop_mask):
        if getattr(self, "_side_stream", None) is None:
            self._side_stream = torch.cuda.Stream()
        sync = self._sync
        # SyncBN: B200SEG_SYNCBN_BRANCH_STREAMS=0 restores the two-chain structure (one stream per scale pass + its side
        # stream, repack on the main stream); the default runs the same 21-stream program as per-GPU statistics - the
        # one-warp waiter kernels never keep another kernel from being scheduled (csrc/bn_kernels.cu), so up to eight
        # exchanges (four branches x two passes) are in flight and hide each other's NVLink round trips.
        import os
        wide = sync is None or os.environ.get("B200SEG_SYNCBN_BRANCH_STREAMS", "1") != "0"
        wd_ready = self._repack(side=self._side_stream if wide else None)
        if sync is not None:
            sync.advance()
        tensors = {k: v.detach() for k, v in self._tensors().items()}
        par = self.parallel_scales and A.is_two_scale(self.arch)
        # (one engine per scale pass, or a single pass: a layer's cells are used once per step)
        use_cells = self.bn_cells and sync is None and (par or not A.is_two_scale(self.arch))
        if use_cells:
            self._bncell_arena.zero_()
        self._acc_hi.zero_()         # two memsets (45 us each) beat clearing inside the fold's transposed gather
        if par:
            self._acc_lo.zero_()
        # every allocation of the step stays referenced until its final join (raw.py)
        raw.KEEP = [] if wide else None
        if getattr(self, "_bstreams", None) is None:
            use_b = self.parallel_branches and wide
            pr = -1 if self._prio() else 0
            mk = lambda: [torch.cuda.Stream(priority=pr) for _ in range(3)] if use_b else []
            self._bstreams = {"hi": mk(), "lo": mk()}
            self._ws_holders = {"hi": [None] if wide else None, "lo": [None] if wide else None}
        grads = self._engine_grads("hi")
        E_lo = None
        if par:
            if getattr(self, "_lo_stream", None) is None:
                self._lo_stream = torch.cuda.Stream(priority=-1 if self._prio() else 0)
                self._side_stream_lo = torch.cuda.Stream()
            grads_lo = self._engine_grads("lo")
            E_lo = Engine(tensors, grads_lo, self._packed, True, drop_mask, side_stream=self._side_stream_lo,
                          bstat=self._bstat_views[0], stream=self._lo_stream, sync=sync, pass_id=0,
                          branch_streams=self._bstreams["lo"], ws_holder=self._ws_holders["lo"],
                          bnfold=self._bnfold[0] if self.fused_bn_finalize else None,
                          bncells=self._bncells[0] if use_cells else None)
        two_pass = A.is_two_scale(self.arch)
        if sync is not None and two_pass and not par:
            raise RuntimeError("SyncBN needs parallel_scales=True for the two-scale step (one engine per pass)")
        E = Engine(tensors, grads, self._packed, True, drop_mask, side_stream=self._side_stream,
                   bstat=self._bstat_views[1] if par else None, sync=sync, pass_id=1 if two_pass else 0,
                   branch_streams=self._bstreams["hi"], ws_holder=self._ws_holders["hi"],
                   bnfold=self._bnfold[1] if self.fused_bn_finalize else None,
                   bncells=self._bncells[1] if use_cells else None)
        loss = M.train_loss(E, images, gts, self.arch, self.hcfg, self.ocfg, self.lo_scale, self.ocr_alpha, self.sup_wt,
                            self.ignore_index, E_lo=E_lo, loss_kind=self.loss_kind)
        E.pre_backward_event = wd_ready
        if E_lo is not None:
            E_lo.pre_backward_event = wd_ready
        bucketed = self._bucketed_allreduce()
        self._reduced_in_step = bucketed
        if bucketed:
            self._run_backward_bucketed(E, E_lo, par)
        else:
            M.run_backward(E, E_lo)
            self._fold_grads(par)
        if par:
            assert E.bn_seen == E_lo.bn_seen and len(E.bn_seen) == len(self._bn_slots), "BN bookkeeping out of sync"
            raw.bn_running_update(self._run_flat, self._bstat[0], self._bstat[1], BN_MOMENTUM, self._nbt_flat, 2)
        raw.KEEP = None
        return loss

    def _bucketed_allreduce(self):
        """Data-parallel step: fold and all-reduce finished gradient buckets while the backward still runs."""
        import os
        # Opt-in (B200SEG_BUCKET_ALLREDUCE=1): NCCL's kernels wait for their peers while holding whole SMs, and every
        # persistent convolution CTA owns its tiles statically - a convolution that shares the GPU with an all-reduce
        # stalls until the collective leaves its SMs, and under SyncBN (compute that waits for the peer's compute) the
        # combination can deadlock, so SyncBN mode never overlaps. Default: one all-reduce at gradient-publish time.
        if not self._ddp_allreduce or self._sync is not None or os.environ.get("B200SEG_BUCKET_ALLREDUCE", "0") != "1":
            return False
        d = torch.distributed
        return d.is_available() and d.is_initialized() and d.get_world_size() > 1

    def _run_backward_bucketed(self, E, E_lo, par):
        """Collective C1 overlapped with the backward (the reference's apex DDP overlaps its buckets the same way,
        network/__init__.py:38-39): when the tapes of all scale passes have passed a bucket's marker, a communication
        stream folds that bucket's accumulators into the step gradient (OIHW) and NCCL all-reduces its slice, while the
        compute streams continue with the earlier layers. Inside the captured graph this is a side branch that joins at
        the end of the step; the 1 / world_size average is applied by the publish kernel."""
        if getattr(self, "_comm_stream", None) is None:
            self._comm_stream = torch.cuda.Stream()
        comm = self._comm_stream
        engines = [E] + ([E_lo] if E_lo is not None else [])
        seen = {}
        works = []
        by_tag = {b["tag"]: b for b in self._buckets}

        def launch(bucket, events):
            with torch.cuda.stream(comm):
                for ev in events:
                    comm.wait_event(ev)
                raw.grad_fold(self._step_flat, self._acc_hi, self._acc_lo if par else None, bucket["table"], clear=False,
                              overwrite=True)
                works.append(torch.distributed.all_reduce(self._step_flat[bucket["lo"]:bucket["hi"]], async_op=True))

        def on_mark(eng, tag):
            if tag not in by_tag:
                return
            cur = torch.cuda.current_stream()
            evs = [cur.record_event()]
            if eng.side is not None:
                evs.append(eng.side.record_event())
            seen.setdefault(tag, []).extend(evs)
            seen[tag + "#n"] = seen.get(tag + "#n", 0) + 1
            if seen[tag + "#n"] == len(engines):
                launch(by_tag[tag], seen[tag])

        for eng in engines:
            eng.on_mark = on_mark
        M.run_backward(E, E_lo)                      # joins every compute stream on the current one at its end
        if "rest" in by_tag:
            launch(by_tag["rest"], [torch.cuda.current_stream().record_event()])
        with torch.cuda.stream(comm):
            for w in works:
                w.wait()
        torch.cuda.current_stream().wait_stream(comm)

    def _drop_mask(self, n, device):
        """Dropout2d(0.05) channel mask (network/ocr_utils.py:146) drawn from torch's generator, folded with 1/(1-p)."""
        if self.is_deepv3:
            # WRN-38 mod6 / mod7: Dropout2d(0.3) / Dropout2d(0.5) in front of conv3 (network/wider_resnet.py:302 patches
            # nn.Dropout to Dropout2d; :336-338). One flat fp32 buffer, [n, c] per block in A.wrn_drop_layout order.
            parts = []
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

    def _train_forward(self, images, gts):
        self._ensure_device_state()
        self._sync_context()
        images = images.contiguous().float()
        gts = gts.contiguous().long()
        key = (tuple(images.shape), str(images.device))
        mask = self._drop_mask(images.shape[0], images.device)
        if not self.use_cuda_graph:
            return self._step_eager(images, gts, mask)
        st = self._graphs.get(key)
        if st is None:
            st = dict(images=images.clone(), gts=gts.clone(), mask=None if mask is None else mask.clone(), calls=0,
                      graph=None, loss=None)
            self._graphs[key] = st
        st["images"].copy_(images)
        st["gts"].copy_(gts)
        if mask is not None:
            st["mask"].copy_(mask)
        st["calls"] += 1
        if st["graph"] is None:
            if st["calls"] < 2:      # first call: eager warm-up (sets kernel attributes, fills the allocator pools)
                return self._step_eager(st["images"], st["gts"], st["mask"])
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                st["loss"] = self._step_eager(st["images"], st["gts"], st["mask"])
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
            if getattr(self, "_reduced_in_step", False):       # the step all-reduced its buckets while it ran
                scale = 1.0 / torch.distributed.get_world_size()
            else:
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
