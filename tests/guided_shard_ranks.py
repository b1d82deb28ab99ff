"""2+ GPUs (torchrun): a frame-sharded handle refuses the guided DDIM update (-1) and `ddim_sample(use_graph=True,
cond_scale != 1)` on a frame-sharded UNet raises NotImplementedError.
   torchrun ... tests/guided_shard_ranks.py"""
import ctypes
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import weights as W            # noqa: E402
from tests import gpu_common as G          # noqa: E402


def main():
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    torch.cuda.set_device(int(os.environ["LOCAL_RANK"]))
    dev = torch.device("cuda", int(os.environ["LOCAL_RANK"]))
    dist.init_process_group("nccl", device_id=dev)
    from dawn_pytorch_b200 import DynamicNfGaussianDiffusion, DynamicNfUnet3D, _lib
    net = DynamicNfUnet3D(**G.CTOR).eval()
    net.load_state_dict(G.synth_sd(), strict=True)
    net = net.to(dev)
    Fl, h, w = 40, 8, 8
    _, fea, cond = W.synth_inputs("guidedshard", Fl * world, h, w)
    net.update_num_frames(Fl)
    net.init_shard(Fl, h, w, dev)
    net.set_clip_invariants(fea[0].to(dev), cond[0, rank * Fl:(rank + 1) * Fl].contiguous().to(dev))
    n = 3 * Fl * h * w
    buf = torch.zeros(2 * n + 512, device=dev)
    p = ctypes.c_void_p(buf.data_ptr())
    rc = _lib.lib.dawn_unet_ddim_step_guided(net._handle, p, p, p, n, p, *[1.0] * 5, 0.9, p,
                                             ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert rc == -1 and b"unsharded" in _lib.lib.dawn_last_error()
    D = DynamicNfGaussianDiffusion(denoise_fn=net, num_frames=40, image_size=32, sampling_timesteps=3, timesteps=1000, loss_type='l2',
                                   use_dynamic_thres=True, null_cond_prob=0.1, ddim_sampling_eta=1.0).to(dev)
    D.update_num_frames(Fl)
    try:
        D.ddim_sample(fea.to(dev), (1, 3, Fl, h, w), cond=cond[:, rank * Fl:(rank + 1) * Fl].contiguous().to(dev), cond_scale=2.0,
                      use_graph=True, seed=0)
        raise AssertionError("guided use_graph on a frame-sharded UNet did not raise")
    except NotImplementedError as e:
        assert "frame-sharded" in str(e)
    if rank == 0:
        print(f"[guided] sharded x{world}: guided step refused, guided graph raises NotImplementedError", flush=True)
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
