"""Executor for the HRNet-OCR-MScale hot path: fused-op forward with an explicit reverse tape.

Design notes
  * Every op is one or a few C-ABI kernel launches (``raw``); there is no per-op autograd graph. The forward pushes
    closures on a tape; ``run_backward`` pops them in reverse. Tapes are static for a given input shape, which is
    what lets ``B200SegModule`` capture the whole fwd+bwd step in one CUDA graph.
  * ``Act`` is an NHWC bf16 activation (possibly a channel-slice view of a wider buffer, so concat is a no-op).
    ``Act.grad`` accumulates in place: producers of a gradient either create it or pass the existing buffer as the
    kernel's addend.
  * conv -> training BatchNorm -> (residual) -> ReLU is three passes: the wgmma conv emits the batch statistics from
    its epilogue, ``bn_finalize`` turns them into scale/shift (+ running stats), ``bn_apply`` fuses affine, residual,
    ReLU and the Dropout2d mask. The backward mirrors it (``bn_bwd`` = reduce + finalize + apply, then wgrad, dgrad).
"""
import contextlib

import torch

from . import raw

BF16 = torch.bfloat16
F32 = torch.float32
BN_EPS = 1e-5
BN_MOMENTUM = 0.1   # network/hrnetv2.py:25 and the nn.BatchNorm2d default


class Act:
    __slots__ = ("t", "grad", "needs_grad", "stats")

    def __init__(self, t, needs_grad=True):
        self.t = t
        self.grad = None
        self.needs_grad = needs_grad
        self.stats = None      # (partials, grid, cpad) batch statistics of t when a pre-activation BatchNorm follows


class ConvBNRec:
    """A convolution + batch-statistics record whose affine/activation is applied later (bn_act or inside a fuse)."""
    __slots__ = ("x", "y", "cname", "bname", "ksize", "stride", "cout", "scale", "shift", "mean", "invstd", "has_bias",
                 "dil", "pending", "par")


class HeadRec:
    """A logit-head convolution (no BN); ``dlogits`` (bf16 [N,h,w,32|8]) is filled in by the loss backward."""
    __slots__ = ("x", "cname", "cout", "logits", "dlogits", "has_bias")


class Engine:
    def __init__(self, params, grads, packed, training, drop_mask=None, side_stream=None, bstat=None, stream=None,
                 sync=None, pass_id=0, branch_streams=None, ws_holder=None, bnfold=None, bncells=None):
        """params: name -> tensor (weights, BN buffers); grads: name -> fp32 tensor accumulated into (training);
        packed: name -> (w_fwd, w_dgrad) bf16 operand caches; drop_mask: fp32 [N, mid] post-ReLU multiplier;
        bstat: BN layer name -> fp32 [2*C] slot receiving the batch [mean | unbiased var] (the running statistics are
        then updated once per step by bn_running_update; without it bn_finalize updates them in place);
        stream: the stream this engine's program is enqueued on when it runs concurrently with another engine (the
        low-resolution pass of the two-scale step), None = the caller's current stream;
        sync / pass_id: SyncBNContext (p2p.py) and this engine's pass index in its exchange table (data parallel);
        bnfold: BN layer name -> (fp64 accumulator, int32 ticket) cells: the BatchNorm statistics are finalised inside
        the convolution launch (raw.conv2d_fwd_bn) instead of by a bn_finalize launch (per-GPU statistics only);
        bncells: BN layer name -> (fp64 forward cells [2*roundup16(c)], fp64 backward cells [2*c]), all zero at the start
        of the step: deferred finalisation - the convolution / the backward reduction only add their sums to the cells
        and the consuming apply pass folds them in its prologue (no finaliser launch on the chain; per-GPU statistics);
        branch_streams: up to three extra streams for the parallel branches of a HighResolutionModule (branch 0 stays
        on the engine's own stream); ws_holder: reusable weight-gradient slab workspace of the side stream."""
        self.p = params
        self.g = grads
        self.packed = packed
        self.training = training
        self.drop_mask = drop_mask
        self.bstat = bstat
        self.stream = stream
        self.sync = sync
        self.pass_id = pass_id
        self.bstreams = list(branch_streams or [])
        self.ws_holder = ws_holder
        self.bnfold = bnfold if sync is None else None
        self.bncells = bncells if (sync is None and self.bnfold is None) else None
        self.eval_bn = None      # evaluation: BN layer name -> (scale, shift) from the running statistics (evalpath.py)
        self._ctx = None         # stream of the branch section being recorded (None = the engine's own stream)
        self.pre_backward_event = None   # e.g. "data-gradient weight operands packed" (recorded on another stream)
        self.tape = []
        self.on_mark = None      # callable(engine, tag): fired in backward when everything recorded after mark(tag) has run
        self.bn_seen = set()
        self.hold = []      # tensors handed across streams: kept alive until the step's final join
        # Weight gradients do not feed the rest of the backward chain: they run on a side stream (a parallel branch of
        # the captured CUDA graph) and overlap with the BN / data-gradient kernels of the main chain.
        self.side = side_stream if side_stream is not None else (
            torch.cuda.Stream() if (training and torch.cuda.is_available()) else None)
        self._keepalive = []

    # ------------------------------------------------------------------------------------------ tape
    def run_backward(self):
        """Pops the tape: ops run on the stream they were recorded on; a forward join becomes a fork and vice versa."""
        tape = self.tape
        if self.pre_backward_event is not None:
            torch.cuda.current_stream().wait_event(self.pre_backward_event)
        while tape:
            kind, fn, st = tape.pop()
            if kind == "op":
                if st is None:
                    fn()
                else:
                    with torch.cuda.stream(st):
                        fn()
            elif kind == "mark":
                if self.on_mark is not None:
                    self.on_mark(self, fn)
            elif kind == "join":          # forward joined k branches here: backward forks them
                self._fork_streams(fn)
            else:                          # forward forked here: backward joins
                self._join_streams(fn)
        if self.side is not None:
            torch.cuda.current_stream().wait_stream(self.side)
        self._keepalive.clear()

    # ------------------------------------------------------------------------------------------ branch sections
    def _fork_streams(self, k):
        base = torch.cuda.current_stream()
        for s in self.bstreams[: k - 1]:
            s.wait_stream(base)

    def _join_streams(self, k):
        base = torch.cuda.current_stream()
        for s in self.bstreams[: k - 1]:
            base.wait_stream(s)

    def fork(self, k):
        """k independent branches follow (HighResolutionModule.branches, network/hrnetv2.py:236-239): branch i > 0 is
        recorded on self.bstreams[i-1], a parallel branch of the captured graph."""
        if not self.bstreams:
            return
        self._fork_streams(k)
        if self.training:
            self.tape.append(("fork", k, None))

    def join(self, k):
        if not self.bstreams:
            return
        self._join_streams(k)
        if self.training:
            self.tape.append(("join", k, None))

    @contextlib.contextmanager
    def on_branch(self, i):
        if i == 0 or not self.bstreams:
            yield
            return
        st = self.bstreams[i - 1]
        prev, self._ctx = self._ctx, st
        try:
            with torch.cuda.stream(st):
                yield
        finally:
            self._ctx = prev

    def mark(self, tag):
        """Checkpoint on the main chain of the program: in backward, on_mark(self, tag) fires once the gradients of
        everything recorded AFTER this point are enqueued (used to hand finished parameter-gradient buckets to the
        data-parallel all-reduce while the rest of the backward still runs)."""
        if self.training:
            self.tape.append(("mark", tag, None))

    def finish(self):
        """After every stream of the step has been joined: drop the cross-stream keep-alive references."""
        self.hold.clear()

    def wgrad(self, x_t, dy, dw, cout, ksize, stride, dilation=1):
        """dw += wgrad(x, dy) on the side stream. Operands are kept alive until the streams are joined (the caching
        allocator must not hand their memory to main-stream allocations while the side stream still reads them)."""
        if self.side is None:
            raw.conv2d_wgrad(x_t, dy, dw, cout, ksize, stride, dilation=dilation)
            return
        main = torch.cuda.current_stream()
        self.side.wait_stream(main)
        with torch.cuda.stream(self.side):
            ws = raw.conv2d_wgrad(x_t, dy, dw, cout, ksize, stride, ws_holder=self.ws_holder, dilation=dilation)
        self._keepalive.append((x_t, dy, ws))

    def _push(self, fn):
        if self.training:
            self.tape.append(("op", fn, self._ctx))

    @staticmethod
    def _accumulate(act, new_grad_fn):
        """new_grad_fn(addend, out) must write out = new (+ addend). Creates act.grad when absent."""
        if act.grad is None:
            act.grad = new_grad_fn(None)
        else:
            new_grad_fn(act.grad)

    # ------------------------------------------------------------------------------------------ conv + BN
    def conv_stats(self, x, cname, bname, ksize, stride=1, bias=False, dilation=1, defer=False):
        """defer: the caller applies the BatchNorm with bn_act right away (conv_bn): with deferred finalisation the
        parameters of the layer exist only once that apply pass has run."""
        w_f, _ = self.packed[cname]
        rec = ConvBNRec()
        rec.x, rec.cname, rec.bname, rec.ksize, rec.stride, rec.has_bias = x, cname, bname, ksize, stride, bias
        rec.cout = w_f.shape[0]
        rec.dil = dilation
        rec.pending = rec.par = None
        b = self.p[cname + ".bias"] if bias else None
        if self.training and defer and self.bncells is not None:
            if self.bstat is not None:
                self.bn_seen.add(bname)
            rec.pending = self.bncells[bname][0]
            rec.y = raw.conv2d_fwd_cells(x.t, w_f, b, stride, rec.pending, dilation=dilation)
            par = rec.par = raw._new((4, rec.cout), dtype=F32, device=x.t.device)
            rec.scale, rec.shift, rec.mean, rec.invstd = par[0], par[1], par[2], par[3]
            return rec
        if self.training and self.bnfold is not None:
            acc, ticket = self.bnfold[bname]
            if self.bstat is not None:
                self.bn_seen.add(bname)
                y, par = raw.conv2d_fwd_bn(x.t, w_f, b, stride, self.p[bname + ".weight"], self.p[bname + ".bias"], BN_EPS,
                                           BN_MOMENTUM, acc, ticket, batch_out=self.bstat[bname], dilation=dilation)
            else:
                y, par = raw.conv2d_fwd_bn(x.t, w_f, b, stride, self.p[bname + ".weight"], self.p[bname + ".bias"], BN_EPS,
                                           BN_MOMENTUM, acc, ticket, running_mean=self.p[bname + ".running_mean"],
                                           running_var=self.p[bname + ".running_var"],
                                           nbt=self.p[bname + ".num_batches_tracked"], dilation=dilation)
            rec.scale, rec.shift, rec.mean, rec.invstd = par[0], par[1], par[2], par[3]
        elif self.training:
            y, stats = raw.conv2d_fwd(x.t, w_f, b, stride=stride, emit_stats=True, dilation=dilation)
            n, ho, wo, _ = y.shape
            if self.bstat is not None:
                self.bn_seen.add(bname)
                par = raw.bn_finalize(stats, n * ho * wo, self.p[bname + ".weight"], self.p[bname + ".bias"], BN_EPS,
                                      BN_MOMENTUM, None, None, None, rec.cout, batch_out=self.bstat[bname],
                                      sync=self._sync(bname, 0))
            else:
                par = raw.bn_finalize(stats, n * ho * wo, self.p[bname + ".weight"], self.p[bname + ".bias"], BN_EPS,
                                      BN_MOMENTUM, self.p[bname + ".running_mean"], self.p[bname + ".running_var"],
                                      self.p[bname + ".num_batches_tracked"], rec.cout, sync=self._sync(bname, 0))
            rec.scale, rec.shift, rec.mean, rec.invstd = par[0], par[1], par[2], par[3]
        else:
            y = raw.conv2d_fwd(x.t, w_f, b, stride=stride, dilation=dilation)
            par = self.eval_bn[bname] if self.eval_bn is not None else raw.bn_eval_params(
                self.p[bname + ".weight"], self.p[bname + ".bias"], BN_EPS, self.p[bname + ".running_mean"],
                self.p[bname + ".running_var"])
            rec.scale, rec.shift, rec.mean, rec.invstd = par[0], par[1], None, None
        rec.y = y
        return rec

    def _sync(self, bname, direction):
        return self.sync.args(self.pass_id, bname, direction) if self.sync is not None else None

    def rec_backward(self, rec, dz, mask, post_scale=None, g_out=None, g_accumulate=False):
        """Backward of BN(conv(x)) given the gradient w.r.t. the BN output (dz, optionally ReLU-masked by `mask`)."""
        dy = raw.bn_bwd(dz, mask, post_scale, rec.y, rec.mean, rec.invstd, self.p[rec.bname + ".weight"],
                        self.g[rec.bname + ".weight"], self.g[rec.bname + ".bias"], g_out=g_out,
                        g_accumulate=g_accumulate, sync=self._sync(rec.bname, 1),
                        fold=self.bnfold[rec.bname] if self.bnfold is not None else None,
                        cells=self.bncells[rec.bname][1] if self.bncells is not None else None)
        x = rec.x
        self.wgrad(x.t, dy, self.g[rec.cname + ".weight"], rec.cout, rec.ksize, rec.stride, rec.dil)
        # a conv bias in front of a training-mode BN has an exactly zero gradient (BN removes the mean): left at 0
        if x.needs_grad:
            _, w_d = self.packed[rec.cname]
            if x.grad is None:
                x.grad = raw.conv2d_dgrad(dy, w_d, tuple(x.t.shape), rec.ksize, rec.stride, dilation=rec.dil)
            else:
                raw.conv2d_dgrad(dy, w_d, tuple(x.t.shape), rec.ksize, rec.stride, addend=x.grad, out=x.grad,
                                 dilation=rec.dil)

    def bn_act(self, rec, relu=True, residual=None, out=None, post_scale=None):
        if rec.pending is not None:       # deferred finalisation: this pass turns the cells into the layer's parameters
            bn = rec.bname
            kw = dict(batch_out=self.bstat[bn]) if self.bstat is not None else dict(
                running_mean=self.p[bn + ".running_mean"], running_var=self.p[bn + ".running_var"],
                nbt=self.p[bn + ".num_batches_tracked"])
            z = raw.bn_apply_cells(rec.y, rec.pending, rec.par, self.p[bn + ".weight"], self.p[bn + ".bias"], BN_EPS,
                                   BN_MOMENTUM, residual.t if residual is not None else None, post_scale, relu, out=out,
                                   **kw)
            rec.pending = None
        else:
            z = raw.bn_apply(rec.y, rec.scale, rec.shift, residual.t if residual is not None else None, post_scale,
                             relu, out=out)
        za = Act(z)

        def bwd():
            dz = za.grad
            if dz is None:
                return   # dead branch (autograd would prune it too)
            g_out, g_acc = None, False
            if residual is not None and residual.needs_grad:
                if residual.grad is None:
                    residual.grad = raw._new(residual.t.shape, dtype=BF16, device=z.device)
                else:
                    g_acc = True
                g_out = residual.grad
            self.rec_backward(rec, dz, z if relu else None, post_scale, g_out, g_acc)
            za.grad = None
        self._push(bwd)
        return za

    def conv_bn(self, x, cname, bname, ksize, stride=1, relu=True, residual=None, out=None, bias=False,
                post_scale=None, dilation=1):
        if not self.training and self.eval_bn is not None and post_scale is None:
            # evaluation: BatchNorm (running statistics), residual sum and ReLU in the convolution epilogue - one launch
            w_f, _ = self.packed[cname]
            scale, shift = self.eval_bn[bname]
            if bias:                 # (conv + b) * s + t = conv * s + (b * s + t)
                shift = shift + self.p[cname + ".bias"].float() * scale
            z = raw.conv2d_fwd_affine(x.t, w_f, scale, shift, relu, stride=stride,
                                      addend=residual.t if residual is not None else None, out=out, dilation=dilation)
            return Act(z)
        rec = self.conv_stats(x, cname, bname, ksize, stride, bias, dilation, defer=True)
        return self.bn_act(rec, relu, residual, out, post_scale)

    # ------------------------------------------------------------------------------------------ pre-activation networks
    def _add_grad(self, act, g):
        """act.grad += g with copy semantics (g may still be read by a weight-gradient kernel on the side stream)."""
        if not act.needs_grad:
            return
        if act.grad is None:
            act.grad = raw._new(g.shape, dtype=BF16, device=g.device)
            raw.masked_accum(g, None, act.grad, False)
        else:
            raw.masked_accum(g, None, act.grad, True)

    def conv_sum(self, x, cname, ksize, stride=1, dilation=1, addend=None, want_stats=False, out=None):
        """y = conv(x) (+ addend) with no normalisation behind it; the epilogue can emit the batch statistics of y for a
        pre-activation BatchNorm further down (IdentityResidualBlock, network/wider_resnet.py:170-183). y may have any
        number of consumers: its producer's backward runs after all of theirs."""
        w_f, _ = self.packed[cname]
        cout = w_f.shape[0]
        stats = None
        res = raw.conv2d_fwd(x.t, w_f, None, stride=stride, emit_stats=want_stats and self.training, dilation=dilation,
                             addend=addend.t if addend is not None else None, out=out)
        if want_stats and self.training:
            y, stats = res
        else:
            y = res
        ya = Act(y)
        ya.stats = stats

        def bwd():
            dy = ya.grad
            if dy is None:
                return
            self.wgrad(x.t, dy, self.g[cname + ".weight"], cout, ksize, stride, dilation)
            if x.needs_grad:
                _, w_d = self.packed[cname]
                if x.grad is None:
                    x.grad = raw.conv2d_dgrad(dy, w_d, tuple(x.t.shape), ksize, stride, dilation=dilation)
                else:
                    raw.conv2d_dgrad(dy, w_d, tuple(x.t.shape), ksize, stride, addend=x.grad, out=x.grad,
                                     dilation=dilation)
            if addend is not None:
                self._add_grad(addend, dy)
            ya.grad = None
        self._push(bwd)
        return ya

    def preact(self, x, bname, post_scale=None):
        """a = relu(BN(x)) for an activation whose batch statistics are already known (x.stats)."""
        c = x.t.shape[3]
        if self.training:
            assert x.stats is not None, "pre-activation BN needs the batch statistics of its input"
            n, h, w, _ = x.t.shape
            par = raw.bn_finalize(x.stats, n * h * w, self.p[bname + ".weight"], self.p[bname + ".bias"], BN_EPS,
                                  BN_MOMENTUM, self.p[bname + ".running_mean"], self.p[bname + ".running_var"],
                                  self.p[bname + ".num_batches_tracked"], c, sync=self._sync(bname, 0))
        elif self.eval_bn is not None:
            par = self.eval_bn[bname]
        else:
            par = raw.bn_eval_params(self.p[bname + ".weight"], self.p[bname + ".bias"], BN_EPS,
                                     self.p[bname + ".running_mean"], self.p[bname + ".running_var"])
        a = raw.bn_apply(x.t, par[0], par[1], None, post_scale, True)
        aa = Act(a)

        def bwd():
            dz = aa.grad
            if dz is None:
                return
            dy = raw.bn_bwd(dz, a, post_scale, x.t, par[2], par[3], self.p[bname + ".weight"],
                            self.g[bname + ".weight"], self.g[bname + ".bias"], sync=self._sync(bname, 1),
                            cells=self.bncells[bname][1] if self.bncells is not None else None)
            if x.needs_grad:
                if x.grad is None:
                    x.grad = dy                  # fresh tensor, no other reader
                else:
                    raw.masked_accum(dy, None, x.grad, True)
            aa.grad = None
        self._push(bwd)
        return aa

    def maxpool(self, x):
        """nn.MaxPool2d(3, 2, 1) (+ the batch statistics of the pooled map for the pre-activation BN behind it)."""
        y = raw.maxpool3x3s2(x.t)
        ya = Act(y)
        if self.training:
            ya.stats = raw.channel_stats(y)

        def bwd():
            if ya.grad is None or not x.needs_grad:
                return
            if x.grad is None:
                x.grad = raw.maxpool3x3s2_bwd(x.t, ya.grad)
            else:
                raw.maxpool3x3s2_bwd(x.t, ya.grad, out=x.grad, accumulate=True)
            ya.grad = None
        self._push(bwd)
        return ya

    def image_pool(self, x):
        """nn.AdaptiveAvgPool2d(1): [n,h,w,c] -> [n,1,1,c]."""
        n, h, w, c = x.t.shape
        va = Act(raw.spatial_sum(x.t, 1.0 / (h * w)))

        def bwd():
            if va.grad is None or not x.needs_grad:
                return
            if x.grad is None:
                x.grad = raw.broadcast_pixels(va.grad, h, w, scale=1.0 / (h * w))
            else:
                raw.broadcast_pixels(va.grad, h, w, out=x.grad, scale=1.0 / (h * w), accumulate=True)
            va.grad = None
        self._push(bwd)
        return va

    def broadcast(self, v, h, w, out):
        """Upsample of a 1x1 map into (a channel slice of) an [n,h,w,*] buffer."""
        oa = Act(raw.broadcast_pixels(v.t, h, w, out=out))

        def bwd():
            if oa.grad is None:
                return
            if v.grad is None:
                v.grad = raw.spatial_sum(oa.grad, 1.0)
            else:
                raw.spatial_sum(oa.grad, 1.0, out=v.grad, accumulate=True)
            oa.grad = None
        self._push(bwd)
        return oa

    # ------------------------------------------------------------------------------------------ fuse / resample
    def fuse(self, out_shape, terms, relu=True, out=None):
        """terms: list of ('id', Act) | ('rec', ConvBNRec) (affine folded in, upsampled when coarser)."""
        n, h, w, c = out_shape
        tl = []
        for kind, obj in terms:
            if kind == "id":
                tl.append((obj.t, None, None))
            else:
                tl.append((obj.y, obj.scale, obj.shift))
        z = raw.fuse_fwd(tl, n, h, w, c, relu, out=out)
        za = Act(z)

        def bwd():
            dz = za.grad
            if dz is None:
                return
            mask = z if relu else None
            for kind, obj in terms:
                if kind == "id":
                    if not obj.needs_grad:
                        continue
                    if obj.t.shape[1] == h and obj.t.shape[2] == w:
                        if obj.grad is None:
                            obj.grad = raw._new(obj.t.shape, dtype=BF16, device=z.device)
                            raw.masked_accum(dz, mask, obj.grad, False)
                        else:
                            raw.masked_accum(dz, mask, obj.grad, True)
                    else:
                        hh, ww = obj.t.shape[1], obj.t.shape[2]
                        if obj.grad is None:
                            obj.grad = raw.upsample_adjoint(dz, mask, hh, ww)
                        else:
                            raw.upsample_adjoint(dz, mask, hh, ww, out=obj.grad, accumulate=True)
                else:
                    yh, yw = obj.y.shape[1], obj.y.shape[2]
                    if yh == h and yw == w:
                        self.rec_backward(obj, dz, mask)
                    else:
                        gl = raw.upsample_adjoint(dz, mask, yh, yw)
                        self.rec_backward(obj, gl, None)
            za.grad = None
        self._push(bwd)
        return za

    def slice_marker(self, parent, pieces):
        """pieces: list of (Act view, c0, c1). In backward, hands each view its slice of parent.grad."""
        def bwd():
            if parent.grad is None:
                return
            for act, c0, c1 in pieces:
                sl = parent.grad[..., c0:c1]
                if act.grad is None:
                    act.grad = sl
                else:   # already has a gradient elsewhere: accumulate into the slice and alias it
                    raw.masked_accum(act.grad, None, sl, True)
                    act.grad = sl
        self._push(bwd)

    # ------------------------------------------------------------------------------------------ logit heads
    def conv_head(self, x, cname, bias=True, ld=20):
        w_f, _ = self.packed[cname]
        cout = w_f.shape[0]
        b = self.p[cname + ".bias"] if bias else None
        logits = raw.conv2d_fwd(x.t, w_f, b, out_fp32=True, out_ld=max(ld, cout))
        rec = HeadRec()
        rec.x, rec.cname, rec.cout, rec.logits, rec.dlogits, rec.has_bias = x, cname, cout, logits, None, bias

        def bwd():
            dl = rec.dlogits
            if dl is None:
                return   # dead head (e.g. the 1x pass' attention, network/ocrnet.py:284-287)
            self.wgrad(x.t, dl, self.g[cname + ".weight"], cout, 1, 1)
            if bias:
                raw.bias_grad(dl, cout, self.g[cname + ".bias"])
            _, w_d = self.packed[cname]
            cpad = w_d.shape[2]
            dlv = dl[..., :cpad]
            if x.grad is None:
                x.grad = raw.conv2d_dgrad(dlv, w_d, tuple(x.t.shape), 1, 1)
            else:
                raw.conv2d_dgrad(dlv, w_d, tuple(x.t.shape), 1, 1, addend=x.grad, out=x.grad)
            rec.dlogits = None
        self._push(bwd)
        return rec
