"""GPU tests of guidance limited to an interval: the cond-only companion's forward against the cond half of the
two-branch forward (bitwise with split-K off, rel L2 with it on) in fp16 and bf16, each sampler over a window of mixed
guided and unguided steps against the host loop with graph replay equal to eager execution, a frame-sharded window on
one GPU (thread-ranks) and over two processes, and FaceAnimatePipeline / ClipAnimator end to end."""
import functools
import json
import os
import subprocess
import sys

import pytest
import torch

from conftest import rel_l2
from test_audio_guidance_cpu import SAMPLERS, _table
from test_guidance_interval_cpu import _host_v
from test_guidance_rescale_cpu import host_update
from test_pipeline_gpu import StubFaceLocator, StubProj, StubReferenceNet, StubVAE, model  # noqa: F401 (fixture)

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


def _window(eng, inp, dev, dtype=torch.float16):
    from hallo_b200.dist import window_inputs_to_device
    eng.begin_window(**window_inputs_to_device(inp, dev, dtype))


def _run(eng, lat0, n):
    eng.latents.copy_(lat0)
    eng.reset_steps()
    for _ in range(n):
        eng.step()
    torch.cuda.synchronize()
    return eng.latents.clone()


@pytest.mark.parametrize("nb", [2, 3])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_cond_only_forward_matches_cond_half(monkeypatch, dtype, nb):
    """16x16, f = 4: the companion's forward (cond rows alone) against the cond rows of the two- or three-branch
    forward.  With split-K off every GEMM / conv row is computed independently of the launch's row count and the
    outputs are bitwise equal.  With the default split-K the row count changes the split of some GEMMs, and the
    random-init UNet amplifies those roundings: measured on an H100, rel L2 1.6e-3 (two branches) and 2.3e-3 (three)
    in fp16, 1.3e-2 and 1.8e-2 in bf16; the bound is 3e-3 in fp16, scaled by bf16's larger unit roundoff.  GroupNorm picks its one-launch or three-launch form by the
    frame count times the frame size (hallo_b200_groupnorm), so the bitwise check uses latents of at most 16x16, where
    every level takes the one-launch form at any frame count; larger latents near that size threshold can round
    differently in the cond-only forward."""
    from hallo_b200 import ops
    from hallo_b200.engine import DenoiseEngine, PackedWeights, Shard
    from hallo_b200.scheduler import DDIMScheduler
    from hallo_b200.spec import UNetConfig
    from hallo_b200.synth import synth_inputs, synth_state_dict_device
    dev = _dev()
    cfg = UNetConfig()
    W = PackedWeights(synth_state_dict_device(cfg, dev, seed=0), cfg, dev, dtype)
    f, size = 4, 16
    inp = synth_inputs(cfg, size, size, f, seed=21)
    eng = DenoiseEngine(W, size, size, f, Shard(halves=tuple(range(nb)), frames=tuple(range(f))))
    _window(eng, inp, dev, dtype)
    d = DDIMScheduler()
    d.set_timesteps(10)
    eng.set_schedule(d.timesteps.tolist(), d.coef_table(), 3.5, audio_guidance=6.0 if nb == 3 else None,
                     guided=[False] * 10)
    cond = eng.cond_engine()
    lat = inp["sample"][:1].float().to(dev)
    split = (rel_l2(cond.forward_only(lat, step=3), eng.forward_only(lat, step=3)[1:2]),)
    for name in ("gemm", "conv3x3", "conv3x3_stride2"):
        monkeypatch.setattr(ops, name, functools.partial(getattr(ops, name), split_k=False))
    full = eng.forward_only(lat, step=3)
    one = cond.forward_only(lat, step=3)
    torch.cuda.synchronize()
    print(f"{dtype}, nb = {nb}: cond-only vs cond half, split-K off: bitwise {torch.equal(one, full[1:2])}; "
          f"split-K on: rel L2 = {split[0]:.2e}")
    assert torch.isfinite(one).all() and one.abs().max() > 0
    assert torch.equal(one, full[1:2])
    assert split[0] <= 3e-3 * torch.finfo(dtype).eps / torch.finfo(torch.float16).eps
    eng.release()


@pytest.mark.parametrize("cls", SAMPLERS, ids=lambda c: c.__name__)
def test_mixed_interval_matches_host_loop(model, cls):
    """16x16, f = 3, 10-step schedule, CFG 3.5, steps 0..4 with steps 1 and 2 guided: the two graphs (main and
    cond-only) against the host loop (forward_only, the float64 combine on guided steps, v_c alone on unguided ones,
    then the sampler's table row); graph replay equals eager execution bitwise; the main graph survives interval
    changes."""
    from hallo_b200.engine import DenoiseEngine, guided_steps
    from hallo_b200.spec import UNetConfig
    from hallo_b200.synth import synth_inputs
    m, _ = model
    dev = _dev()
    f, n, steps = 3, 10, 5
    inp = synth_inputs(UNetConfig(), 16, 16, f, seed=5)
    lat0 = inp["sample"][:1].float().to(dev)
    ts, kind, table = _table(cls, n)
    mask = guided_steps(ts, (ts[2], ts[1]))
    assert mask[:steps] == [False, True, True, False, False]
    noise = (torch.randn(n, 4, f, 16, 16, generator=torch.Generator().manual_seed(3)).to(dev, torch.float16)
             if kind == "ancestral" else None)
    eng = DenoiseEngine(m._weights(), 16, 16, f)
    _window(eng, inp, dev)
    eng.set_schedule(ts, table, 3.5, kind, noise=noise)
    x, state = lat0.double(), {}
    for i in range(steps):
        mo = eng.forward_only(x.float(), step=i).double()
        v = _host_v(mo, 2, 3.5, 0.0, 0.0, mask[i])
        x = host_update(kind, table[i], x, v, state, None if noise is None else noise[i].double().unsqueeze(0))
    eng.capture()
    g = eng.graph
    plain = _run(eng, lat0, steps)
    eng.set_schedule(ts, table, 3.5, kind, noise=noise, guided=mask)
    cond = eng.cond_engine()
    cond.capture()
    assert eng.graph is g and cond.graph is not None
    graph = _run(eng, lat0, steps)
    gc = cond.graph
    eng.graph = cond.graph = None
    eager = _run(eng, lat0, steps)
    eng.graph, cond.graph = g, gc
    err, moved = rel_l2(graph, x), rel_l2(plain, graph)
    print(f"{cls.__name__}, {steps} of {n} steps, 2 guided: graphs vs host loop rel L2 = {err:.2e}; "
          f"graph == eager: {torch.equal(graph, eager)}; every step guided vs interval: {moved:.2e}")
    assert torch.isfinite(graph).all() and err < 1e-2 and moved > 5 * err
    assert torch.equal(graph, eager)
    eng.release()


def test_frame_sharded_window_matches_unsharded(model, monkeypatch):
    """Two ranks as threads on one GPU (conftest.ThreadGroup, the engine's exchange="nccl" path), four eager
    DPM-Solver++ steps with steps 1 and 2 guided: the gathered latents equal the unsharded engine's."""
    from conftest import ThreadGroup
    from hallo_b200.dist import shard_layout
    from hallo_b200.engine import DenoiseEngine, Shard
    from hallo_b200.spec import UNetConfig
    from hallo_b200.synth import synth_inputs
    m, _ = model
    dev = _dev()
    f, R, size, steps = 16, 2, 32, 4
    inp = synth_inputs(UNetConfig(), size, size, f, seed=42)
    W = m._weights()
    ts, kind, table = _table(SAMPLERS[1], 10)
    mask = [i in (1, 2) for i in range(10)]
    lat0 = inp["sample"][:1].float().to(dev)
    full = DenoiseEngine(W, size, size, f)
    _window(full, inp, dev)
    full.set_schedule(ts, table, 3.5, kind, guided=mask)
    ref = _run(full, lat0, steps)
    full.set_schedule(ts, table, 3.5, kind)
    plain = _run(full, lat0, steps)
    full.release()
    del full
    grp = ThreadGroup(R, monkeypatch)
    layout = shard_layout(R, f)

    def rank_fn(r):
        torch.cuda.set_device(dev)
        halves, frames = layout[r]
        eng = DenoiseEngine(W, size, size, f, Shard(halves=halves, frames=frames, group=grp, group_size=R,
                                                    rank_in_group=r, exchange="nccl"))
        _window(eng, inp, dev)
        eng.set_schedule(ts, table, 3.5, kind, guided=mask)
        out = _run(eng, lat0[:, :, list(frames)], steps)
        eng.release()
        return out

    got = torch.cat(grp.run(rank_fn), dim=2)
    err, moved = rel_l2(got, ref), rel_l2(plain, ref)
    print(f"{R} thread-ranks vs unsharded, {steps} DPM-Solver++ steps, 2 guided: rel L2 = {err:.2e} "
          f"(every step guided vs interval: {moved:.2e})")
    assert err < 5e-3 and moved > 5 * err


@pytest.mark.parametrize("exchange", ["peer", "nccl"])
def test_two_process_sharded_window_with_interval(exchange):
    """tests/mgpu_interval_worker.py under torchrun on two GPUs (skipped on fewer): a frame-sharded window with
    guided and unguided steps against the unsharded engine, eager and graph."""
    n = torch.cuda.device_count() if torch.cuda.is_available() else 0
    if n < 2:
        pytest.skip("needs >= 2 CUDA devices")
    port = 29543 if exchange == "peer" else 29544
    env = dict(os.environ, HALLO_B200_EXCHANGE=exchange, MASTER_ADDR="127.0.0.1", SIZE="32", FRAMES="16")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
                        "--master-addr", "127.0.0.1", "--master-port", str(port),
                        os.path.join(ROOT, "tests", "mgpu_interval_worker.py")],
                       env=env, capture_output=True, text=True, timeout=900)
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("MGPU_RESULT ")]
    assert r.returncode == 0 and lines, r.stdout[-3000:] + r.stderr[-3000:]
    res = json.loads(lines[-1][len("MGPU_RESULT "):])
    print(res)
    assert all(c == 0 for c in res["device_errors_all_ranks"]), res
    assert res["eager_rel_l2"] < 5e-3 and res["graph_rel_l2"] < 5e-3, res


def _pipe(m, dev, H, W):
    from hallo_b200.animate.face_animate import FaceAnimatePipeline
    from hallo_b200.scheduler import DDIMScheduler
    sched = DDIMScheduler(beta_start=0.00085, beta_end=0.012, beta_schedule="linear", clip_sample=False, steps_offset=1,
                          prediction_type="v_prediction", rescale_betas_zero_snr=True, timestep_spacing="trailing")
    pipe = FaceAnimatePipeline(vae=StubVAE(), reference_unet=StubReferenceNet(H // 8, W // 8), denoising_unet=m,
                               face_locator=StubFaceLocator((1,)), scheduler=sched, image_proj=StubProj((1, 4, 768)))
    return pipe.to(device=dev, dtype=torch.float16)


def test_face_animate_pipeline_guidance_interval(model):
    """128x128, f = 4, 8 DDIM steps (timesteps 999, 874, ..., 124), CFG 3.5: an interval that holds every step gives
    the video of a call without the keyword bitwise, through the same engine and graph and without a companion; an
    interval holding some steps changes the video, keeps the main graph, and with a callback gives the same video and
    the callback every step's latents in the usual form."""
    m, _ = model
    dev = _dev()
    H = W = 128
    f, n = 4, 8
    pipe = _pipe(m, dev, H, W)
    gen = torch.Generator().manual_seed(7)
    masks = [torch.rand(f, ((H // 8) // s) * ((W // 8) // s), generator=gen) for s in (1, 2, 4, 8)]
    ref_image = torch.rand(1, 3, 3, H, W, generator=gen) * 2 - 1
    face_emb = torch.randn(1, 512, generator=gen)
    audio = torch.randn(1, f, 32, 768, generator=gen).to(dev, torch.float16)
    face_mask = torch.rand(1, 3, H, W, generator=gen)

    def call(**kw):
        return pipe(ref_image=ref_image, face_emb=face_emb, audio_tensor=audio, face_mask=face_mask,
                    pixel_values_full_mask=masks, pixel_values_face_mask=masks, pixel_values_lip_mask=masks, width=W,
                    height=H, video_length=f, num_inference_steps=n, guidance_scale=3.5,
                    generator=torch.Generator().manual_seed(9), motion_scale=[1.0, 1.0, 1.0], **kw).videos

    v_default = call()
    eng = m.engine(H // 8, W // 8, f)
    g = eng.graph
    v_all = call(guidance_interval=(0, 1000))
    assert m.engine(H // 8, W // 8, f) is eng and eng.graph is g and eng._cond is None
    seen = []
    v_mid = call(guidance_interval=(300, 700))
    assert eng.guided is not None and sum(eng.guided) == 3 and eng.graph is g and eng._cond.graph is not None
    v_mid_eager = call(guidance_interval=(300, 700), callback=lambda i, t, x: seen.append((i, tuple(x.shape))))
    v_default2 = call()
    e_mid = rel_l2(v_mid, v_default)
    print(f"pipeline, {n} DDIM steps: interval over every step vs no keyword bitwise {torch.equal(v_all, v_default)}; "
          f"3 guided steps vs every step {e_mid:.2e}; with a callback {torch.equal(v_mid, v_mid_eager)}")
    assert torch.equal(v_all, v_default) and torch.equal(v_default2, v_default)
    assert torch.isfinite(v_mid).all() and e_mid > 1e-3 and tuple(v_mid.shape) == (1, 3, f, H, W)
    assert torch.equal(v_mid, v_mid_eager)
    assert seen == [(i, (1, 4, f, H // 8, W // 8)) for i in range(n)]


def test_clip_animator_guidance_interval(model):
    """Two 4-frame windows with the motion-frame hand-off, 4 DDIM steps: an interval over every step gives the clip of
    no keyword bitwise; an interval holding some steps changes it and stays finite."""
    from hallo_b200.driver import ClipAnimator, process_audio_emb
    from hallo_b200.models.audio_proj import AudioProjModel
    m, _ = model
    dev = _dev()
    H = W = 128
    cl = 4
    pipe = _pipe(m, dev, H, W)
    torch.manual_seed(0)
    ap = AudioProjModel().to(dev, torch.float16)
    gen = torch.Generator().manual_seed(17)
    masks = [torch.rand(1, ((H // 8) // s) * ((W // 8) // s), generator=gen) for s in (1, 2, 4, 8)]
    audio = process_audio_emb(torch.randn(2 * cl, 12, 768, generator=gen))
    args = dict(source_image_pixels=torch.rand(3, H, W, generator=gen) * 2 - 1,
                source_image_face_region=torch.rand(3, H, W, generator=gen),
                source_image_face_emb=torch.randn(512, generator=gen), source_image_full_mask=masks,
                source_image_face_mask=masks, source_image_lip_mask=masks, audio_emb=audio, width=W, height=H,
                num_inference_steps=4, guidance_scale=3.5)
    anim = ClipAnimator(pipe, ap, clip_length=cl, n_motion_frames=2)
    v_none = anim(**args, generator=torch.manual_seed(42))
    v_all = anim(**args, generator=torch.manual_seed(42), guidance_interval=(-1, 1e4))
    v_mid = anim(**args, generator=torch.manual_seed(42), guidance_interval=(500, 1000))
    err = rel_l2(v_mid, v_none)
    print(f"clip driver: interval over every step vs none bitwise {torch.equal(v_all, v_none)}; "
          f"interval (500, 1000) vs none {err:.2e}")
    assert torch.equal(v_all, v_none)
    assert torch.isfinite(v_mid).all() and err > 1e-3
