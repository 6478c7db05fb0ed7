"""GPU tests of the UniPC sampler: the hallo_b200_cfg_unipc_step kernel against float64 in fp16 and bf16, the
engine's UniPC loop (host loop, graph replay, capture in mid-schedule, window restart, switching back to DDIM),
FaceAnimatePipeline with the stand-in scheduler, and a frame-sharded window on two GPUs."""
import json
import os
import subprocess
import sys

import pytest
import torch

from conftest import rel_l2
from test_pipeline_gpu import StubFaceLocator, StubProj, StubReferenceNet, StubVAE, model  # noqa: F401 (fixture)

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U = 2.0 ** -24                                               # fp32 unit roundoff


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_cfg_unipc_kernel_matches_float64(dtype):
    """5 chained steps through the device counter, the whole 5-step schedule: row 0 without corrector (NaN-filled
    state), row 1 with the order-1 corrector, rows 2-3 with the order-2 corrector and a second-order predictor, and
    the final row onto sigma = 0.  ldm = 8 > Cl = 4 with NaN in the unused columns, F * HW = 189 (not a multiple of
    the 128-thread block).  Bound, per element: 16 u times the sum of the magnitudes of every term (u = 2^-24), for
    the latents, the corrected sample and the data estimate; each step's reference starts from the device's state."""
    from hallo_b200 import ops
    from hallo_b200.scheduler import UniPCMultistepScheduler
    dev = _dev()
    cl, f, h, w, ldm, g_s, n = 4, 3, 7, 9, 8, 3.5, 5
    n_tok = f * h * w
    s = UniPCMultistepScheduler()
    s.set_timesteps(n)
    coef = s.coef_table().to(dev)
    c64 = coef.double().cpu()
    assert c64[0, 2] == 1 and c64[1, 2] == 0 and c64[1, 6] == 0 and c64[2, 6] != 0 and c64[2, 9] != 0
    assert c64[4, 7] == 0 and c64[4, 9] == 0                 # row 4: sigma_5 = 0, first order
    gen = torch.Generator().manual_seed(21)
    lat = torch.randn(1, cl, f, h, w, generator=gen).to(dev)
    state = [torch.full_like(lat, float("nan")) for _ in range(3)]      # last_sample, x0_hist, x0_hist2
    step = torch.zeros(1, dtype=torch.int32, device=dev)
    worst = 0.0
    for i in range(n):
        # this step's inputs: the device state as it stands (fp32, exact in float64); NaN where not yet written
        x, last, m1, m2 = [t.double().cpu() for t in [lat] + state]
        mo = torch.full((2 * n_tok, ldm), float("nan"))
        mo[:, :cl] = torch.randn(2 * n_tok, cl, generator=gen)
        mo = mo.to(dev, dtype)
        ops.cfg_unipc_step(mo, lat, *state, coef, step, guidance=g_s)
        ops.advance_step(step, n)
        torch.cuda.synchronize()
        mm = mo.double().cpu()[:, :cl]

        def bcfhw(t):
            return t.reshape(f, h, w, cl).permute(3, 0, 1, 2).unsqueeze(0)
        vu, vc = bcfhw(mm[:n_tok]), bcfhw(mm[n_tok:])
        v = vu + g_s * (vc - vu)
        al, sg, kx, kl, k0, k1, k2, pc, p0, p1 = c64[i].tolist()
        m = al * x - sg * v
        m_mag = (al * x).abs() + abs(sg) * (vu.abs() + g_s * (vc - vu).abs())
        c, c_mag = k0 * m, abs(k0) * m_mag
        for k, t in ((kx, x), (kl, last), (k1, m1), (k2, m2)):
            if k != 0.0:
                c, c_mag = c + k * t, c_mag + (k * t).abs()
        xn = pc * c + p0 * m + (p1 * m1 if p1 != 0.0 else 0.0)
        x_mag = abs(pc) * c_mag + abs(p0) * m_mag + ((p1 * m1).abs() if p1 != 0.0 else 0.0)
        for g, want, mag in zip([lat, state[0], state[1]], (xn, c, m), (x_mag, c_mag, m_mag)):
            g = g.double().cpu()
            assert torch.isfinite(g).all(), i
            ratio = float(((g - want).abs() / (U * mag + 1e-30)).max())
            worst = max(worst, ratio)
            assert ratio <= 16.0, (i, ratio)
        assert torch.equal(state[2].double().cpu().nan_to_num(7.0), m1.nan_to_num(7.0)), i     # x0_hist2 <- x0_hist
    print(f"{dtype}: worst error / (u * term magnitude) = {worst:.2f} (bound 16)")
    assert int(step) == 0                                    # the counter wrapped: the next window starts at row 0


def _engine_window(eng, inp, dev, dt):
    from hallo_b200.dist import window_inputs_to_device
    eng.begin_window(**window_inputs_to_device(inp, dev, dt))


def _reset(eng, lat0, nan_state=False):
    eng.latents.copy_(lat0)
    eng.step_idx.zero_()
    if nan_state:
        for buf in (eng.last_sample, eng.x0_hist, eng.x0_hist2):
            buf.fill_(float("nan"))


def _run(eng, lat0, n, nan_state=False):
    _reset(eng, lat0, nan_state)
    for _ in range(n):
        eng.step()
    torch.cuda.synchronize()
    return eng.latents.clone()


def test_engine_unipc_loop(model):
    """16x16, f = 3, a 10-step UniPC bh2 schedule, CFG 3.5."""
    from hallo_b200.engine import DenoiseEngine
    from hallo_b200.scheduler import DDIMScheduler, UniPCMultistepScheduler, sampler_table_of
    from hallo_b200.spec import UNetConfig
    from hallo_b200.synth import synth_inputs
    m, _ = model
    dev, dt = _dev(), torch.float16
    inp = synth_inputs(UNetConfig(), 16, 16, 3, seed=5, motion_scale=(1.0, 1.0, 1.0))
    lat0 = inp["sample"][:1].float().to(dev)
    eng = m.engine(16, 16, 3)
    _engine_window(eng, inp, dev, dt)
    s = UniPCMultistepScheduler()
    s.set_timesteps(10)
    kind, table = sampler_table_of(s)
    assert kind == "unipc"
    ts = s.timesteps.tolist()
    # host loop: the engine's UNet forward, CFG and the scheduler's own float64 step() on the host
    eng.set_schedule(ts, table, 3.5, kind)
    x = lat0.clone()
    for i, t in enumerate(ts[:6]):
        mo = eng.forward_only(x, step=i)
        x = s.step(mo[:1] + 3.5 * (mo[1:] - mo[:1]), t, x).prev_sample
    eng.set_schedule(ts, table, 3.5, kind)
    eng.graph = None
    _reset(eng, lat0, nan_state=True)
    eng.capture()
    g_uni = eng.graph
    graph6 = _run(eng, lat0, 6, nan_state=True)
    err = rel_l2(graph6, x)
    print(f"6 of 10 UniPC bh2 steps: graph vs host loop rel L2 = {err:.3e}")
    assert int(eng.step_idx) == 6 and torch.isfinite(graph6).all() and err < 1e-2
    # graph replay == eager execution of the same plan
    eng.graph = None
    eager6 = _run(eng, lat0, 6, nan_state=True)
    print(f"graph vs eager rel L2 = {rel_l2(graph6, eager6):.3e}")
    assert torch.equal(graph6, eager6)
    # a capture after 3 eager steps keeps the latents, the counter and all three state buffers across its warm-up
    _run(eng, lat0, 3, nan_state=True)
    eng.capture()
    for _ in range(3):
        eng.step()
    torch.cuda.synchronize()
    assert int(eng.step_idx) == 6 and torch.equal(eng.latents, eager6)
    eng.graph = g_uni
    # two whole windows through the same graph: the second starts on row 0 over the first's stale state
    w1 = _run(eng, lat0, 10)
    assert int(eng.step_idx) == 0
    eng.latents.copy_(lat0)
    for _ in range(10):
        eng.step()
    torch.cuda.synchronize()
    assert eng.graph is g_uni and torch.isfinite(w1).all() and torch.equal(eng.latents, w1)
    # back to DDIM on the same engine: the graph is dropped and the result equals a fresh engine's
    d = DDIMScheduler()
    d.set_timesteps(10)
    eng.set_schedule(d.timesteps.tolist(), d.coef_table(), 3.5)
    assert eng.graph is None
    eng.capture()
    ddim_same = _run(eng, lat0, 3)
    fresh = DenoiseEngine(eng.W, 16, 16, 3)
    _engine_window(fresh, inp, dev, dt)
    fresh.set_schedule(d.timesteps.tolist(), d.coef_table(), 3.5)
    fresh.capture()
    ddim_fresh = _run(fresh, lat0, 3)
    assert torch.equal(ddim_same, ddim_fresh) and not torch.equal(ddim_same, lat0)
    del fresh


@pytest.mark.parametrize("steps", [10, 20])
def test_face_animate_pipeline_with_unipc(model, steps):
    from hallo_b200.animate.face_animate import FaceAnimatePipeline
    from hallo_b200.scheduler import UniPCMultistepScheduler
    m, _ = model
    dev = _dev()
    H = W = 128
    f = 4
    sched = UniPCMultistepScheduler(beta_start=0.00085, beta_end=0.012, beta_schedule="linear", clip_sample=False,
                                    steps_offset=1, prediction_type="v_prediction", rescale_betas_zero_snr=True,
                                    timestep_spacing="trailing")
    pipe = FaceAnimatePipeline(vae=StubVAE(), reference_unet=StubReferenceNet(H // 8, W // 8), denoising_unet=m,
                               face_locator=StubFaceLocator((1,)), scheduler=sched, image_proj=StubProj((1, 4, 768)))
    pipe.to(device=dev, dtype=torch.float16)
    gen = torch.Generator().manual_seed(7)
    masks = [torch.rand(f, ((H // 8) // s) * ((W // 8) // s), generator=gen) for s in (1, 2, 4, 8)]
    ref_image = torch.rand(1, 3, 3, H, W, generator=gen) * 2 - 1
    face_emb = torch.randn(1, 512, generator=gen)
    audio = torch.randn(1, f, 32, 768, generator=gen).to(dev, torch.float16)
    face_mask = torch.rand(1, 3, H, W, generator=gen)
    eng = m.engine(H // 8, W // 8, f)

    def call(use_graph, callback=None):
        pipe.use_cuda_graph = use_graph
        if not use_graph:
            eng.graph = None
        return pipe(ref_image=ref_image, face_emb=face_emb, audio_tensor=audio, face_mask=face_mask,
                    pixel_values_full_mask=masks, pixel_values_face_mask=masks, pixel_values_lip_mask=masks, width=W,
                    height=H, video_length=f, num_inference_steps=steps, guidance_scale=3.5,
                    generator=torch.Generator().manual_seed(9), motion_scale=[1.0, 1.0, 1.0], callback=callback,
                    callback_steps=1).videos

    v_graph = call(True)
    assert eng.graph is not None and eng.sampler == "unipc" and pipe.last_timing["steps"] == steps
    v_eager = call(False)
    seen = []
    v_cb = call(False, callback=lambda i, t, lat: seen.append((i, int(t), lat.clone())))
    assert tuple(v_graph.shape) == (1, 3, f, H, W) and torch.isfinite(v_graph).all()
    err, err_cb = rel_l2(v_graph, v_eager), rel_l2(v_cb, v_eager)
    print(f"pipeline, {steps} UniPC steps: graph vs eager rel L2 = {err:.3e}, callback run vs eager = {err_cb:.3e}")
    assert err < 1e-3 and err_cb < 1e-3
    ts = sched.timesteps.tolist()
    assert [(i, t) for i, t, _ in seen] == [(i, ts[i]) for i in range(steps)]
    assert all(tuple(lat.shape) == (1, 4, f, H // 8, W // 8) and torch.isfinite(lat).all() for _, _, lat in seen)
    # callbacks receive s_{i+1}, what diffusers' step() returns: the last one is the window's final latents
    assert torch.equal(seen[-1][2], eng.latents.to(seen[-1][2].dtype))
    assert not torch.equal(seen[-2][2], seen[-1][2])


WORKER = r'''
import json, os, sys
import torch
import torch.distributed as dist
sys.path.insert(0, os.environ["HB_ROOT"])
rank, world, lr = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
torch.cuda.set_device(lr)
dev = torch.device("cuda", lr)
dist.init_process_group("nccl", device_id=dev)
from hallo_b200 import lib
from hallo_b200.dist import plan_shard, sharded_vs_unsharded, window_inputs_to_device
from hallo_b200.engine import DenoiseEngine, PackedWeights
from hallo_b200.scheduler import UniPCMultistepScheduler, sampler_table_of
from hallo_b200.spec import UNetConfig
from hallo_b200.synth import synth_inputs, synth_state_dict_device
cfg = UNetConfig()
W = PackedWeights(synth_state_dict_device(cfg, dev, seed=0), cfg, dev, torch.float16)
inp = synth_inputs(cfg, 32, 32, 16, seed=42)
sh = plan_shard(rank, world, 16)
eng = DenoiseEngine(W, 32, 32, 16, sh)
eng.begin_window(**window_inputs_to_device(inp, dev, torch.float16))
s = UniPCMultistepScheduler()
s.set_timesteps(10)
kind, table = sampler_table_of(s)
eng.set_schedule(s.timesteps.tolist(), table, 3.5, kind)
res = {"eager_rel_l2": sharded_vs_unsharded(eng, inp, steps=4)}
eng.latents.copy_(inp["sample"][:1, :, list(sh.frames)].float().to(dev))
eng.capture()
res["graph_rel_l2"] = sharded_vs_unsharded(eng, inp, steps=4, use_graph=True)
res["device_error"] = lib.device_error()
if rank == 0:
    print("UNI_RESULT " + json.dumps(res), flush=True)
eng.graph = None
torch.cuda.synchronize()
if eng.arena is not None:
    eng.arena.close()
dist.barrier()
sys.stdout.flush()
os._exit(0)
'''


def test_frame_sharded_unipc_matches_unsharded(tmp_path):
    """Two ranks: the unipc kind and table reach sharded_vs_unsharded's unsharded engine; 4 steps (the order-2
    corrector from step 2 on), eagerly and through the graph, within tests/test_multigpu_gpu.py's 5e-3."""
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 CUDA devices")
    script = tmp_path / "uni_worker.py"
    script.write_text(WORKER)
    env = dict(os.environ, HB_ROOT=ROOT, MASTER_ADDR="127.0.0.1")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
                        "--master-addr", "127.0.0.1", "--master-port", "29543", str(script)],
                       env=env, capture_output=True, text=True, timeout=900)
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("UNI_RESULT ")]
    assert r.returncode == 0 and lines, r.stdout[-3000:] + r.stderr[-3000:]
    res = json.loads(lines[-1][len("UNI_RESULT "):])
    print(res)
    assert res["device_error"] == 0 and res["eager_rel_l2"] < 5e-3 and res["graph_rel_l2"] < 5e-3, res
