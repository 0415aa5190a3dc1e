"""Data-parallel SyncBN step of archs 'basic.HRNet_ASP' and 'mscale.HRNet_ASP' on 2 GPUs of one node against the
single-GPU step on the concatenated batch, within the bounds of tests/test_gpu_multi.py. Narrow test trunk. Skipped on
boxes with fewer than two GPUs."""
import os
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _worker(rank, world, port, out, arch):
    import torch.distributed as dist
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")
    os.environ.setdefault("CUDA_MODULE_LOADING", "EAGER")     # no lazy kernel loading while a GPU spins on its peer
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", init_method="env://", rank=rank, world_size=world)
    import _hrnet_asp_oracle as HA
    from oracle import seg_oracle as O
    from b200seg.module import B200SegModule
    sd0 = HA.synth_state_dict(arch, O.HRNET_W16_TEST, seed=3)
    images, gts = O.synth_batch(world, 128, 256, seed=5)

    def run(batch_slice, ddp):
        net = B200SegModule(arch, 19, hcfg=O.HRNET_W16_TEST, use_cuda_graph=True, syncbn=ddp)
        net.load_state_dict(sd0)
        net = net.cuda().train()
        net._ddp_allreduce = ddp
        losses = []
        for _ in range(3):                        # eager warm-up, capture, replay
            net.zero_grad(set_to_none=True)
            loss = net({"images": images[batch_slice].cuda(), "gts": gts[batch_slice].cuda()})
            loss.backward()
            losses.append(loss.detach().clone())
        torch.cuda.synchronize()
        return net, torch.stack(losses)

    net, losses = run(slice(rank, rank + 1), True)
    dist.all_reduce(losses)
    losses /= world
    if rank == 0:
        ref, ref_losses = run(slice(0, world), False)
        rel = lambda a, b: float((a.double() - b.double()).norm() / (b.double().norm() + 1e-30))
        torch.save(dict(loss=losses.cpu().tolist(), ref_loss=ref_losses.cpu().tolist(),
                        grad_rel=rel(net._flat_grad, ref._flat_grad), run_rel=rel(net._run_flat, ref._run_flat),
                        nbt=(int(net._nbt_flat[0]), int(ref._nbt_flat[0]))), out)
    dist.barrier()
    if net._sync is not None:
        net._sync.close()
    dist.destroy_process_group()


@pytest.mark.timeout(420)
@pytest.mark.parametrize("arch", ["basic.HRNet_ASP", "mscale.HRNet_ASP"])
def test_two_gpu_syncbn_step_equals_single_gpu_batch(tmp_path, arch):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    out = str(tmp_path / "res.pt")
    port = 29500 + (os.getpid() % 1000) + (13 if arch == "basic.HRNet_ASP" else 17)
    mp.spawn(_worker, args=(2, port, out, arch), nprocs=2, join=True)
    res = torch.load(out)
    for a, b in zip(res["loss"], res["ref_loss"]):
        assert abs(a - b) <= 2e-3 * abs(b), res
    assert res["run_rel"] <= 2e-3, res
    assert res["grad_rel"] <= 0.05, res
    assert res["nbt"][0] == res["nbt"][1]
