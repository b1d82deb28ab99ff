"""2+ GPUs (torchrun): the ancestral (DDPM) sampler on a frame-sharded clip vs the single-GPU sampler, same seed.
   torchrun ... tests/ddpm_shard_ranks.py [eager] [graph]     (default: both)"""
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import weights as W            # noqa: E402
from tests import gpu_common as G          # noqa: E402

T = 6                                       # a 6-step schedule: every step of the loop, t = 0 included


def main():
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    torch.cuda.set_device(int(os.environ["LOCAL_RANK"]))
    dev = torch.device("cuda", int(os.environ["LOCAL_RANK"]))
    dist.init_process_group("nccl", device_id=dev)
    from dawn_pytorch_b200 import DynamicNfGaussianDiffusion, DynamicNfUnet3D

    def make(F):
        net = DynamicNfUnet3D(**G.CTOR).eval()
        net.load_state_dict(G.synth_sd(), strict=True)
        D = DynamicNfGaussianDiffusion(denoise_fn=net.to(dev), num_frames=40, image_size=32, sampling_timesteps=None, timesteps=T,
                                       loss_type='l2', use_dynamic_thres=True, null_cond_prob=0.1, ddim_sampling_eta=1.0).to(dev)
        D.update_num_frames(F)
        return D

    Fg, h, w = 48 * world, 16, 16
    Fl, lo = Fg // world, rank * (Fg // world)
    _, fea, cond = W.synth_inputs("shardddpm", Fg, h, w)
    D = make(Fl)
    D.denoise_fn.update_num_frames(Fl)
    D.denoise_fn.init_shard(Fl, h, w, dev)
    assert D.denoise_fn.shard_info() == (rank, world)
    one = None
    if rank == 0:
        D1 = make(Fg)
        one = D1.p_sample_loop(fea.to(dev), (1, 3, Fg, h, w), cond=cond.to(dev), seed=123)[0].cpu()
        del D1
    dist.barrier()
    modes = [m for m in ("eager", "graph") if m in (set(sys.argv[1:]) or {"eager", "graph"})]
    for mode in modes:
        out = D.p_sample_loop(fea.to(dev), (1, 3, Fl, h, w), cond=cond[:, lo:lo + Fl].contiguous().to(dev), seed=123,
                              use_graph=(mode == "graph"))[0].clone()
        parts = [torch.empty_like(out) for _ in range(world)]
        dist.all_gather(parts, out)
        if rank == 0:
            full = torch.cat(parts, dim=1).cpu()
            dmax = (full - one).abs().max().item()
            print(f"[ddpm] F={Fg} sharded x{world} ancestral loop ({mode}), {T} steps: max|d| vs single-GPU {dmax:.2e}", flush=True)
            assert dmax < 2e-4, "sharded ancestral sampler disagrees with the single-GPU sampler"
        dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
