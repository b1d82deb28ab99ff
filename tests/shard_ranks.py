"""2+ GPUs (torchrun): exact frame sharding of one clip vs the reference golden / the unsharded CUDA path.
   torchrun ... tests/shard_ranks.py [forward] [ddim] [ddim_graph]     (default: forward ddim)"""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import weights as W            # noqa: E402
from tests import gpu_common as G          # noqa: E402


def sampler_case(net, rank, world, dev, graph_modes):
    """Row a16 under sharding: 3 DDIM steps (first, middle, last of the 20-step schedule) on a frame-sharded clip — clip-wide
    quantile through all-reduced radix select, per-rank slice of one clip-wide noise tensor — vs the single-GPU sampler."""
    from dawn_pytorch_b200 import DynamicNfGaussianDiffusion, DynamicNfUnet3D
    Fg, h, w = 48 * world, 16, 16
    Fl, lo = Fg // world, rank * (Fg // world)
    x_t, fea, cond = W.synth_inputs("shardddim", Fg, h, w)

    def make(unet):
        return DynamicNfGaussianDiffusion(denoise_fn=unet, num_frames=40, image_size=32, sampling_timesteps=20, timesteps=1000,
                                          loss_type='l2', use_dynamic_thres=True, null_cond_prob=0.1, ddim_sampling_eta=1.0).to(dev)
    D = make(net)
    sched = D.ddim_schedule()
    pairs = [sched[0], sched[10], sched[-1]]

    def noise_global(k):
        return x_t[0] if k < 0 else torch.from_numpy(W.pseudo_normal(f"shardddim/noise{k}", (3, Fg, h, w)))

    net.update_num_frames(Fl)
    net.init_shard(Fl, h, w, dev)
    assert net.shard_info() == (rank, world)
    D.update_num_frames(Fl)
    for use_graph in graph_modes:
        out = D.ddim_sample(fea.to(dev), (1, 3, Fl, h, w), cond=cond[:, lo:lo + Fl].contiguous().to(dev), pairs=pairs,
                            noise_fn=lambda k, shp: noise_global(k)[:, lo:lo + Fl].reshape(shp).clone(), use_graph=use_graph)[0].clone()
        parts = [torch.empty_like(out) for _ in range(world)]
        dist.all_gather(parts, out)
        full = torch.cat(parts, dim=1).cpu()
        if rank == 0:
            net1 = DynamicNfUnet3D(**G.CTOR).eval()
            net1.load_state_dict(G.synth_sd(), strict=True)
            D1 = make(net1.to(dev))
            D1.update_num_frames(Fg)
            one = D1.ddim_sample(fea.to(dev), (1, 3, Fg, h, w), cond=cond.to(dev), pairs=pairs,
                                 noise_fn=lambda k, shp: noise_global(k).reshape(shp).clone())[0].cpu()
            dmax = (full - one).abs().max().item()
            print(f"[ddim] F={Fg} sharded x{world} sampler ({'graph' if use_graph else 'eager'}), 3 steps: max|d| vs single-GPU {dmax:.2e}",
                  flush=True)
            assert dmax < 2e-4, "sharded sampler disagrees with the single-GPU sampler"
            del D1, net1
        dist.barrier()
    # default noise: one clip-wide stream, sliced per rank
    a = D.ddim_sample(fea.to(dev), (1, 3, Fl, h, w), cond=cond[:, lo:lo + Fl].contiguous().to(dev), pairs=pairs[:2], seed=123)
    assert torch.isfinite(a).all()


def main():
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    torch.cuda.set_device(int(os.environ["LOCAL_RANK"]))
    dev = torch.device("cuda", int(os.environ["LOCAL_RANK"]))
    dist.init_process_group("nccl", device_id=dev)
    from dawn_pytorch_b200 import DynamicNfUnet3D
    net = DynamicNfUnet3D(**G.CTOR).eval()
    net.load_state_dict(G.synth_sd(), strict=True)
    net = net.to(dev)
    what = set(sys.argv[1:]) or {"forward", "ddim"}
    cases = [("band", 96, 8, 8, 952, True), ("shardbig", 80 * world, 32, 32, 500, False)] if "forward" in what else []
    for name, Fg, h, w, t, has_golden in cases:
        if Fg % world or Fg // world < 40:
            continue
        Fl, lo = Fg // world, rank * (Fg // world)
        x_t, fea, cond = W.synth_inputs(name, Fg, h, w)
        tt = torch.full((1,), t, dtype=torch.long, device=dev)
        net.update_num_frames(Fl)
        net.init_shard(Fl, h, w, dev)
        net.set_clip_invariants(fea[0].to(dev), cond[0, lo:lo + Fl].contiguous().to(dev))
        out = net.forward_x3(x_t[0, :, lo:lo + Fl].contiguous().to(dev), tt).clone()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize(); dist.barrier(); e0.record()
        for _ in range(3):
            net.forward_x3(x_t[0, :, lo:lo + Fl].contiguous().to(dev), tt)
        e1.record(); torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / 3
        # a parameter re-commit drops the sharding; init_shard on every rank restores it, on the GroupNorm mailboxes the first
        # init_shard allocated, and the sharded forward then returns the same eps (to the last bits the GroupNorm statistics'
        # atomics leave to chance)
        net.load_state_dict(G.synth_sd(), strict=True)
        net.init_shard(Fl, h, w, dev)
        net.set_clip_invariants(fea[0].to(dev), cond[0, lo:lo + Fl].contiguous().to(dev))
        again = net.forward_x3(x_t[0, :, lo:lo + Fl].contiguous().to(dev), tt)
        print(f"[{name}] rank {rank}: sharded forward after a re-commit and init_shard: max|d| {(again - out).abs().max():.2e}",
              flush=True)
        assert (again - out).abs().max().item() <= 1e-5, "the sharded forward changed after a re-commit and init_shard"
        parts = [torch.empty_like(out) for _ in range(world)]
        dist.all_gather(parts, out)
        full = torch.cat(parts, dim=1).cpu()[None]
        if rank == 0:
            if has_golden:
                ref = torch.from_numpy(G.golden(name)["eps"])
                r = G.over_tol(full, ref)
                print(f"[{name}] sharded x{world} vs reference golden: over_tol {r:.3f}", flush=True)
                assert r <= 1.0, "sharded forward disagrees with the reference golden"
            # unsharded run of the whole clip on rank 0 with a second module instance
            net1 = DynamicNfUnet3D(**G.CTOR).eval()
            net1.load_state_dict(G.synth_sd(), strict=True)
            net1 = net1.to(dev)
            net1.update_num_frames(Fg)
            net1.set_clip_invariants(fea[0].to(dev), cond[0].to(dev))
            one = net1.forward_x3(x_t[0].to(dev), tt)
            torch.cuda.synchronize()
            r1 = G.over_tol(full, one.cpu()[None])
            print(f"[{name}] F={Fg} {h}x{w}: sharded x{world} vs single-GPU CUDA: over_tol {r1:.4f}"
                  f"  max|d| {(full[0] - one.cpu()).abs().max():.2e};  sharded step {ms:.2f} ms", flush=True)
            assert r1 <= 0.25, "sharded forward disagrees with the single-GPU forward"
            del net1
        dist.barrier()
    modes = ([False] if "ddim" in what else []) + ([True] if "ddim_graph" in what else [])
    if modes:
        sampler_case(net, rank, world, dev, modes)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
