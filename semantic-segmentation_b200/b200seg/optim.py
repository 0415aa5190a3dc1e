"""FusedSGD: torch.optim.SGD semantics (the optimizer loss/optimizer.py:43-60 builds for every script) with ONE kernel
launch per parameter group instead of torch's foreach chains (SURVEY.md §8(f) row f3). Drop-in: same constructor
arguments, same ``param_groups`` (LR schedulers keep working), momentum buffers exposed as
``state[p]['momentum_buffer']`` views of one flat buffer per group."""
import numpy as np
import torch

from ._lib import check, lib, ptr, stream_ptr


class FusedSGD(torch.optim.Optimizer):
    def __init__(self, params, lr=1e-3, momentum=0.0, dampening=0.0, weight_decay=0.0, nesterov=False):
        if nesterov and (momentum <= 0 or dampening != 0):
            raise ValueError("Nesterov momentum requires a momentum and zero dampening")
        super().__init__(params, dict(lr=lr, momentum=momentum, dampening=dampening, weight_decay=weight_decay,
                                      nesterov=nesterov))
        self._tables = {}

    def _table(self, gi, group):
        ps = [p for p in group["params"] if p.grad is not None]
        key = tuple((p.data_ptr(), p.grad.data_ptr()) for p in ps)
        tab = self._tables.get(gi)
        if tab is not None and tab["key"] == key:
            return tab
        dev = ps[0].device
        total = sum((p.numel() + 63) // 64 * 64 for p in ps)
        old = {id(p): self.state[p]["momentum_buffer"].clone() for p in ps if "momentum_buffer" in self.state.get(p, {})}
        flat = torch.zeros(total, dtype=torch.float32, device=dev)
        chunk = lib().b200seg_sgd_chunk()
        # blocks of the parameters without a momentum buffer come first: their first update starts the buffer at the
        # gradient (torch.optim.SGD), whatever buffers the group's other parameters already hold
        items, blocks = [], ([], [])
        off = 0
        for i, p in enumerate(ps):
            assert p.is_cuda and p.dtype == torch.float32 and p.is_contiguous() and p.grad.is_contiguous()
            buf = flat[off:off + p.numel()].view_as(p)
            if id(p) in old:
                buf.copy_(old[id(p)])
            self.state[p]["momentum_buffer"] = buf
            items.append((p.data_ptr(), p.grad.data_ptr(), buf.data_ptr(), p.numel()))
            blocks[id(p) in old].extend((i, st) for st in range(0, p.numel(), chunk))
            off += (p.numel() + 63) // 64 * 64
        blk_item = [i for i, _st in blocks[0] + blocks[1]]
        blk_start = [st for _i, st in blocks[0] + blocks[1]]
        it_np = np.array(items, dtype=np.dtype([("p", "<u8"), ("g", "<u8"), ("m", "<u8"), ("n", "<i8")]))
        tab = dict(key=key, items=torch.from_numpy(it_np.view(np.uint8).copy()).to(dev),
                   blk_item=torch.tensor(blk_item, dtype=torch.int32, device=dev),
                   blk_start=torch.tensor(blk_start, dtype=torch.int32, device=dev), n_blocks=len(blk_item),
                   n_fresh=len(blocks[0]), flat=flat)
        self._tables[gi] = tab
        return tab

    @torch.no_grad()
    def step(self, closure=None):
        loss = closure() if closure is not None else None
        for gi, group in enumerate(self.param_groups):
            if not any(p.grad is not None for p in group["params"]):
                continue
            tab = self._table(gi, group)
            nf = tab["n_fresh"]
            for first, lo, hi in ((1, 0, nf), (0, nf, tab["n_blocks"])):
                if hi > lo:
                    check(lib().b200seg_sgd_step(ptr(tab["items"]), ptr(tab["blk_item"][lo:]), ptr(tab["blk_start"][lo:]),
                                                 hi - lo, float(group["lr"]), float(group["momentum"]),
                                                 float(group["dampening"]), float(group["weight_decay"]),
                                                 int(group["nesterov"]), first, stream_ptr()), "sgd_step")
            tab["n_fresh"] = 0
        return loss
