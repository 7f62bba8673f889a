"""TEST INFRASTRUCTURE: one rank of a world-size-2 gloo dry run of the DDPO epoch driver with ``--lora_rank 4`` on the
CPU ops emulator (spawned by tests/test_lora_cpu.py).  Usage: python _lora_driver_worker.py <rank> <world> <port> <out>"""
import os
import sys

rank, world, port, out_dir = int(sys.argv[1]), int(sys.argv[2]), sys.argv[3], sys.argv[4]
os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=port, RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK="0")
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
os.chdir(out_dir)

import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

import _lora_emulator as E  # noqa: E402
from ddpo_b200 import unet as U, unet_spec, utils, vae as V  # noqa: E402
from ddpo_b200.diffusers_patch import pipeline_stable_diffusion as P, scheduling_ddim as SD  # noqa: E402
from ddpo_b200.pipeline import policy_gradient as DRV  # noqa: E402
from ddpo_b200.training import policy_gradient as PG  # noqa: E402

for mod in (U, V, P, SD, PG, DRV):
    mod.ops = E
U.Arena = V.Arena = E.CpuArena
PG.USE_CUDA_GRAPH = False
_init = P.StableDiffusionPipeline.__init__


def _no_graph(self, *a, **k):
    k["use_cuda_graph"] = False
    _init(self, *a, **k)


P.StableDiffusionPipeline.__init__ = _no_graph
torch.set_num_threads(2)
dist.init_process_group("gloo", rank=rank, world_size=world)
try:
    models = utils.load_unet(None, pretrained_model="tiny", device="cpu", seed=0, text_encoder="stub")
    argv = ["--dataset", "compressed_animals", "--pretrained_model", "tiny", "--resolution", "128",
            "--sample_batch_size", "2", "--num_sample_batches_per_epoch", "1", "--n_inference_steps", "2",
            "--train_batch_size", "2", "--train_macro", "2", "--num_train_epochs", "2", "--save_freq", "1",
            "--learning_rate", "1e-3", "--savepath", "run_lora", "--seed", "3", "--lora_rank", "4"]
    out = DRV.main(argv, models=models, max_epochs=2)
    net = models[0].unet
    dist.barrier()
    tree = utils.restore_checkpoint(os.path.join("logs/compressed-animals/run_lora", "checkpoints"))
    rewards = np.load(os.path.join(out["localpath"], f"rewards/{rank}_0.npy"))
    np.savez(os.path.join(out_dir, f"lora_rank{rank}.npz"), adapters=out["state"].params.numpy(),
             step=out["state"].step, rewards=rewards, unet=net.params.numpy(), merged=net.merged_params().numpy(),
             checkpoint=utils.flat_from_tree(tree, unet_spec.TINY).numpy())
finally:
    dist.destroy_process_group()
