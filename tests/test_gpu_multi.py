"""Data-parallel step on 2 GPUs of one node (SURVEY.md §8e). Skipped on boxes with fewer than two GPUs.

  * default data-parallel mode (BatchNorm statistics local to each GPU, ONE NCCL all-reduce over the flat gradient
    buffer): every rank must end up with the mean of the per-rank gradients;
  * SyncBN mode (opt-in, `syncbn=True`): statistics exchanged through NVLink peer memory inside the BN finalisers must
    reproduce the single-GPU step on the concatenated batch. That test passed on 2 GPUs at commit 05390e9; later
    multi-stream changes were not re-validated, so it only runs with B200SEG_TEST_SYNCBN=1."""
import os

import pytest
import torch

pytestmark = pytest.mark.gpu


def _worker(rank, world, port, use_graph, out):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")
    os.environ.setdefault("CUDA_MODULE_LOADING", "EAGER")     # no lazy kernel loading while a GPU spins on its peer
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", init_method="env://", rank=rank, world_size=world)
    from oracle import seg_oracle as O
    from b200seg.module import B200SegModule
    arch, hcfg = "ocrnet.HRNet_Mscale", O.HRNET_W16_TEST
    sd0 = O.synth_state_dict(arch, hcfg, seed=3)
    images, gts = O.synth_batch(world, 64, 128, seed=5)
    ocfg = dict(O.OCR_CFG)
    ocfg["dropout"] = 0.0

    def run(batch_slice, ddp, steps):
        net = B200SegModule(arch, 19, hcfg=hcfg, ocfg=ocfg, use_cuda_graph=use_graph, syncbn=ddp)
        net.load_state_dict(sd0)
        net = net.cuda().train()
        net._ddp_allreduce = ddp
        im, gt = images[batch_slice].cuda(), gts[batch_slice].cuda()
        losses = []
        for _ in range(steps):
            net.zero_grad(set_to_none=True)
            loss = net({"images": im, "gts": gt})
            loss.backward()
            losses.append(loss.detach().clone())
        torch.cuda.synchronize()
        return net, torch.stack(losses)

    steps = 3                                   # eager warm-up, capture, replay
    net, losses = run(slice(rank, rank + 1), True, steps)
    dist.all_reduce(losses)
    losses /= world
    if rank == 0:
        ref, ref_losses = run(slice(0, world), False, steps)      # one GPU, whole batch, local BN == SyncBN over ranks
        rel = lambda a, b: float((a.double() - b.double()).norm() / (b.double().norm() + 1e-30))
        res = dict(loss=losses.cpu().tolist(), ref_loss=ref_losses.cpu().tolist(),
                   grad_rel=rel(net._flat_grad, ref._flat_grad),
                   run_rel=rel(net._run_flat, ref._run_flat),
                   nbt=(int(net._nbt_flat[0]), int(ref._nbt_flat[0])))
        torch.save(res, out)
    dist.barrier()
    if net._sync is not None:
        net._sync.close()
    dist.destroy_process_group()


def _ddp_worker(rank, world, port, out):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", init_method="env://", rank=rank, world_size=world)
    from oracle import seg_oracle as O
    from b200seg.module import B200SegModule
    arch, hcfg = "ocrnet.HRNet_Mscale", O.HRNET_W16_TEST
    sd0 = O.synth_state_dict(arch, hcfg, seed=3)
    images, gts = O.synth_batch(world, 64, 128, seed=5)
    ocfg = dict(O.OCR_CFG)
    ocfg["dropout"] = 0.0

    def run(i, ddp):
        net = B200SegModule(arch, 19, hcfg=hcfg, ocfg=ocfg, use_cuda_graph=True)
        net.load_state_dict(sd0)
        net = net.cuda().train()
        net._ddp_allreduce = ddp
        for _ in range(3):                        # eager warm-up, capture, replay
            net.zero_grad(set_to_none=True)
            loss = net({"images": images[i:i + 1].cuda(), "gts": gts[i:i + 1].cuda()})
            loss.backward()
        torch.cuda.synchronize()
        return net._flat_grad.clone(), float(loss)

    g, loss = run(rank, True)
    if rank == 0:
        singles = [run(i, False) for i in range(world)]
        mean = sum(s[0] for s in singles) / world
        rel = float((g.double() - mean.double()).norm() / (mean.double().norm() + 1e-30))
        torch.save(dict(rel=rel, loss=loss, loss_single=singles[0][1]), out)
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.timeout(300)
def test_two_gpu_data_parallel_gradients_are_the_rank_mean(tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    out = str(tmp_path / "ddp.pt")
    port = 29500 + (os.getpid() % 1000) + 7
    mp.spawn(_ddp_worker, args=(2, port, out), nprocs=2, join=True)
    res = torch.load(out)
    assert res["rel"] <= 1e-5, res               # same kernels on the same data; only the all-reduce's sum order differs
    assert abs(res["loss"] - res["loss_single"]) <= 1e-6 * abs(res["loss_single"]), res


@pytest.mark.timeout(420)
@pytest.mark.parametrize("use_graph", [False, True])
def test_two_gpu_syncbn_step_equals_single_gpu_batch(tmp_path, use_graph):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    out = str(tmp_path / "res.pt")
    port = 29500 + (os.getpid() % 1000) + (1 if use_graph else 0)
    mp.spawn(_worker, args=(2, port, use_graph, out), nprocs=2, join=True)
    res = torch.load(out)
    for a, b in zip(res["loss"], res["ref_loss"]):
        assert abs(a - b) <= 2e-3 * abs(b), res
    assert res["run_rel"] <= 2e-3, res          # running statistics come from the global batch
    assert res["grad_rel"] <= 0.05, res         # bf16 activations, different reduction order across the two layouts
    assert res["nbt"][0] == res["nbt"][1]
