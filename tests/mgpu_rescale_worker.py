"""torchrun worker of tests/test_guidance_rescale_gpu.py (one process per GPU): a frame-sharded DenoiseEngine with
guidance rescale (phi = 0.7) against the unsharded engine, eagerly and through the captured CUDA graph, for the exchange
named by HALLO_B200_EXCHANGE.  Also checks that every rank holds bitwise-equal window totals (so applies the same
factor).  Prints one line `MGPU_RESULT {json}` on rank 0."""
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
from hallo_b200.scheduler import DDIMScheduler  # noqa: E402
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
sch = DDIMScheduler()
sch.set_timesteps(40)
eng.set_schedule(sch.timesteps.tolist(), sch.coef_table(), 3.5, guidance_rescale=0.7)
res = {"world": world, "exchange": sh.exchange, "size": size, "frames": f, "guidance_rescale": 0.7}
res["eager_rel_l2"] = sharded_vs_unsharded(eng, inp, steps=2)


def totals():
    t = (eng.arena.local("rescale", (world, 4), torch.float64) if eng.arena is not None
         else eng._bufs[("rescale.totals", world, 4, torch.float64)])
    every = [torch.empty_like(t) for _ in range(world)]
    dist.all_gather(every, t.clone(), group=sh.group)
    return all(torch.equal(every[0], x) for x in every)


res["totals_equal_eager"] = totals()
eng.latents.copy_(inp["sample"][:1, :, list(sh.frames)].float().to(dev))
eng.capture()
res["graph_rel_l2"] = sharded_vs_unsharded(eng, inp, steps=2, use_graph=True)
res["totals_equal_graph"] = totals()
res["device_error"] = lib.device_error()
codes = [None] * world
dist.all_gather_object(codes, res["device_error"])
res["device_errors_all_ranks"] = codes
if rank == 0:
    print("MGPU_RESULT " + json.dumps(res), flush=True)
eng.graph = None
torch.cuda.synchronize()
if eng.arena is not None:
    eng.arena.close()
dist.barrier()
if sh.exchange == "nccl":      # a process that captured NCCL work into a CUDA graph cannot destroy its group promptly
    sys.stdout.flush()
    os._exit(0)
dist.destroy_process_group()
faulthandler.cancel_dump_traceback_later()
