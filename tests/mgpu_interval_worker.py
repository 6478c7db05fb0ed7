"""torchrun worker of tests/test_guidance_interval_gpu.py (one process per GPU): a frame-sharded DenoiseEngine whose
schedule has guided and unguided steps (the unguided ones run the cond-only companion, with its own frame <-> pixel
exchange) against the unsharded engine, eagerly and through the captured CUDA graphs, for the exchange named by
HALLO_B200_EXCHANGE.  Prints one line `MGPU_RESULT {json}` on rank 0."""
import faulthandler
import json
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
faulthandler.dump_traceback_later(int(os.environ.get("WATCHDOG", 240)), repeat=False, exit=True)

rank, world, lr = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
torch.cuda.set_device(lr)
dev = torch.device("cuda", lr)
dist.init_process_group("nccl", device_id=dev)

from hallo_b200 import lib  # noqa: E402
from hallo_b200.dist import plan_shard, sharded_vs_unsharded, window_inputs_to_device  # noqa: E402
from hallo_b200.engine import DenoiseEngine, PackedWeights  # noqa: E402
from hallo_b200.scheduler import DPMSolverMultistepScheduler, sampler_table_of  # noqa: E402
from hallo_b200.spec import UNetConfig  # noqa: E402
from hallo_b200.synth import host_threads, synth_inputs, synth_state_dict_device  # noqa: E402

torch.set_num_threads(max(1, host_threads() // world))
cfg = UNetConfig()
size, f = int(os.environ.get("SIZE", 32)), int(os.environ.get("FRAMES", 16))
W = PackedWeights(synth_state_dict_device(cfg, dev, seed=0), cfg, dev, torch.float16)
inp = synth_inputs(cfg, size, size, f, seed=42)
sh = plan_shard(rank, world, f)
eng = DenoiseEngine(W, size, size, f, sh)
eng.begin_window(**window_inputs_to_device(inp, dev, torch.float16))
sch = DPMSolverMultistepScheduler()
sch.set_timesteps(40)
kind, table = sampler_table_of(sch)
mask = [i in (1, 2) for i in range(40)]
eng.set_schedule(sch.timesteps.tolist(), table, 3.5, kind, guided=mask)
res = {"world": world, "exchange": sh.exchange, "size": size, "frames": f, "guided": [i for i in range(4) if mask[i]]}
res["eager_rel_l2"] = sharded_vs_unsharded(eng, inp, steps=4)
eng.latents.copy_(inp["sample"][:1, :, list(sh.frames)].float().to(dev))
eng.capture()
eng.cond_engine().capture()
res["graph_rel_l2"] = sharded_vs_unsharded(eng, inp, steps=4, use_graph=True)
res["device_error"] = lib.device_error()
codes = [None] * world
dist.all_gather_object(codes, res["device_error"])
res["device_errors_all_ranks"] = codes
if rank == 0:
    print("MGPU_RESULT " + json.dumps(res), flush=True)
torch.cuda.synchronize()
eng.release()
dist.barrier()
if sh.exchange == "nccl":      # a process that captured NCCL work into a CUDA graph cannot destroy its group promptly
    sys.stdout.flush()
    os._exit(0)
dist.destroy_process_group()
faulthandler.cancel_dump_traceback_later()
