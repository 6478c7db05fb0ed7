"""GPU tests of guidance rescale: the three kernels (stats, reduce, apply) against float64 rescale_noise_cfg in fp16
and bf16, their properties and run-to-run bitwise equality, each sampler on the engine against the host loop with
graph replay equal to eager execution, a frame-sharded window on one GPU (thread-ranks) and over two processes (peer
arena), and FaceAnimatePipeline end to end."""
import ctypes as C
import json
import os
import subprocess
import sys

import pytest
import torch

from conftest import rel_l2
from test_audio_guidance_cpu import SAMPLERS, _table
from test_guidance_rescale_cpu import (_halves, check_properties, combine_f64, host_update, make_model_out,
                                       rescale_factor, rescale_noise_cfg_f64, run_rescale, to_bcfhw)
from test_pipeline_gpu import StubFaceLocator, StubProj, StubReferenceNet, StubVAE, model  # noqa: F401 (fixture)

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


@pytest.mark.parametrize("shape", [(3, 7, 9), (2, 200, 201)], ids=["F3xHW63", "F2xHW40200"])
@pytest.mark.parametrize("nb", [2, 3])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_rescale_kernels_match_float64(dtype, nb, shape):
    """ldm = 8 > Cl = 4 with NaN past Cl; F * HW = 189 (one partial CTA) or 80400 (more rows than the 256 x 256
    threads of the stats grid, not a multiple of either block); |v| up to about 1e3.  The cond rows get the rescaled v
    rounded once to the model dtype, the uncond rows 0; a second launch gives bitwise-equal output."""
    from hallo_b200 import ops
    dev = _dev()
    cl, ldm, s, sa, phi = 4, 8, 3.5, 6.0, 0.7
    f, h, w = shape
    n = f * h * w
    mo = make_model_out(nb, cl, f, h * w, ldm, dtype, scale=300.0, device=dev)
    ref = mo.clone().cpu()
    again = mo.clone()
    tot = run_rescale(ops, mo, nb=nb, cl=cl, frames=f, hw=h * w, guidance=s, audio_guidance=sa, rescale=phi)
    tot2 = run_rescale(ops, again, nb=nb, cl=cl, frames=f, hw=h * w, guidance=s, audio_guidance=sa, rescale=phi)
    torch.cuda.synchronize()
    halves = [to_bcfhw(x, cl, f, h, w) for x in _halves(ref, nb, cl, n)]
    vcfg = combine_f64(torch.cat(halves), nb, s, sa)
    want = rescale_noise_cfg_f64(vcfg, halves[1], phi)
    got = to_bcfhw(mo[n:2 * n, :cl].cpu(), cl, f, h, w).double()
    err = float((got - want).abs().max() / want.abs().max())
    k = rescale_factor(tot.cpu(), cl * n, phi)
    print(f"cfg_rescale nb={nb} {dtype} F*HW={n}: max error / max |v| = {err:.2e} (unit roundoff "
          f"{torch.finfo(dtype).eps / 2:.1e}); factor {k:.6f}")
    assert err <= torch.finfo(dtype).eps / 2 + 8 * torch.finfo(torch.float32).eps
    assert abs(k - 1.0) > 1e-2
    assert torch.equal(mo.nan_to_num(), again.nan_to_num())
    assert torch.equal(tot, tot2)
    got_all = mo.cpu()
    assert torch.equal(got_all[:n, :cl].float(), torch.zeros(n, cl)) and got_all[:, cl:].isnan().all()
    if nb == 3:
        assert torch.equal(got_all[2 * n:, :cl], ref[2 * n:, :cl])


def test_rescale_entry_points_validate():
    from hallo_b200 import lib
    dev = _dev()
    h_ = lib.load()
    stream = lib.current_stream()
    mo = torch.zeros(2 * 64, 8, device=dev, dtype=torch.float16)
    part = torch.zeros(256, 4, device=dev, dtype=torch.float64)
    tot = torch.zeros(2, 4, device=dev, dtype=torch.float64)
    f16 = C.c_int(lib.dtype_code(torch.float16))
    P = lambda t: C.c_void_p(None if t is None else t.data_ptr())                   # noqa: E731

    def stats(dt=f16, m=mo, ldm=8, nb=2, cl=4, p=part):
        return h_.hallo_b200_cfg_rescale_stats(dt, P(m), C.c_int64(ldm), C.c_int(nb), C.c_float(3.5), C.c_float(0.0),
                                               C.c_int(cl), C.c_int(1), C.c_int(64), P(p), stream)

    def apply(dt=f16, m=mo, ldm=8, nb=2, cl=4, t=tot, ranks=2, phi=0.7):
        return h_.hallo_b200_cfg_rescale_apply(dt, P(m), C.c_int64(ldm), C.c_int(nb), C.c_float(3.5), C.c_float(0.0),
                                               C.c_float(phi), P(t), C.c_int(ranks), C.c_int(cl), C.c_int(1),
                                               C.c_int(64), stream)

    def reduce(p=part, dst=(tot[0], tot[1]), n=None):
        arr = (C.c_void_p * max(1, len(dst)))(*[P(d) for d in dst])
        return h_.hallo_b200_cfg_rescale_reduce(P(p), arr, C.c_int(len(dst) if n is None else n), stream)

    assert stats() == 0 and reduce() == 0 and apply() == 0
    for bad in (dict(m=None), dict(p=None), dict(dt=C.c_int(7)), dict(ldm=2), dict(nb=4), dict(nb=1), dict(cl=0)):
        assert stats(**bad) != 0, bad
    for bad in (dict(m=None), dict(t=None), dict(dt=C.c_int(7)), dict(ldm=2), dict(nb=4), dict(ranks=0),
                dict(ranks=17), dict(phi=1.5), dict(phi=float("nan"))):
        assert apply(**bad) != 0, bad
    for bad in (dict(p=None), dict(dst=(None,)), dict(n=0), dict(n=17)):
        assert reduce(**bad) != 0, bad
    torch.cuda.synchronize()


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_rescale_kernel_properties(dtype):
    """phi = 1: std of the written v equals std(v_c) to the dtype's rounding; phi = 0: v_cfg itself (and, for three
    branches, exactly guide3's output); a constant v_cfg is kept, not NaN."""
    from hallo_b200 import ops
    err = check_properties(ops, dtype, device=_dev())
    print(f"{dtype}: phi = 1, |std(v) / std(v_c) - 1| = {err:.2e}")


def _window(eng, inp, dev):
    from hallo_b200.dist import window_inputs_to_device
    eng.begin_window(**window_inputs_to_device(inp, dev, torch.float16))


def _run(eng, lat0, n):
    eng.latents.copy_(lat0)
    eng.step_idx.zero_()
    for _ in range(n):
        eng.step()
    torch.cuda.synchronize()
    return eng.latents.clone()


@pytest.mark.parametrize("cls", SAMPLERS, ids=lambda c: c.__name__)
def test_engine_with_rescale_matches_host_loop(model, cls):
    """16x16, f = 3, 10-step schedule, CFG 3.5, phi = 0.7: 4 steps through the CUDA graph against the host loop
    (the engine's forward_only, float64 combine, float64 rescale_noise_cfg and the sampler's table row); graph replay
    equals eager execution bitwise; phi = 0 lands far from phi = 0.7."""
    from hallo_b200.engine import DenoiseEngine
    from hallo_b200.spec import UNetConfig
    from hallo_b200.synth import synth_inputs
    m, _ = model
    dev = _dev()
    f, n, steps = 3, 10, 4
    inp = synth_inputs(UNetConfig(), 16, 16, f, seed=5)
    lat0 = inp["sample"][:1].float().to(dev)
    ts, kind, table = _table(cls, n)
    noise = (torch.randn(n, 4, f, 16, 16, generator=torch.Generator().manual_seed(3)).to(dev, torch.float16)
             if kind == "ancestral" else None)
    eng = DenoiseEngine(m._weights(), 16, 16, f)
    _window(eng, inp, dev)
    eng.set_schedule(ts, table, 3.5, kind, noise=noise, guidance_rescale=0.7)
    x, state = lat0.double(), {}
    for i in range(steps):
        mo = eng.forward_only(x.float(), step=i).double()
        v = rescale_noise_cfg_f64(combine_f64(mo, 2, 3.5, 0.0), mo[1:2], 0.7)
        x = host_update(kind, table[i], x, v, state, None if noise is None else noise[i].double().unsqueeze(0))
    eng.set_schedule(ts, table, 3.5, kind, noise=noise, guidance_rescale=0.7)
    eng.capture()
    graph = _run(eng, lat0, steps)
    g = eng.graph
    eng.graph = None
    eager = _run(eng, lat0, steps)
    eng.graph = g
    eng.set_schedule(ts, table, 3.5, kind, noise=noise)
    assert eng.graph is None                                    # phi is part of the graph key
    plain = _run(eng, lat0, steps)
    err, moved = rel_l2(graph, x), rel_l2(plain, graph)
    print(f"{cls.__name__}, {steps} of {n} steps at phi = 0.7: graph vs host loop rel L2 = {err:.2e}; "
          f"graph == eager: {torch.equal(graph, eager)}; phi = 0 vs 0.7: {moved:.2e}")
    assert torch.isfinite(graph).all() and err < 1e-2 and moved > 5 * err
    assert torch.equal(graph, eager)
    del eng


def test_frame_sharded_window_with_rescale_matches_unsharded(model, monkeypatch):
    """Two ranks as threads on one GPU (conftest.ThreadGroup, the engine's exchange="nccl" path), three eager DDIM
    steps at phi = 0.7: the gathered latents equal the unsharded engine's, and both ranks hold bitwise-equal totals."""
    from conftest import ThreadGroup
    from hallo_b200.dist import shard_layout
    from hallo_b200.engine import DenoiseEngine, Shard
    from hallo_b200.scheduler import DDIMScheduler
    from hallo_b200.spec import UNetConfig
    from hallo_b200.synth import synth_inputs
    m, _ = model
    dev = _dev()
    f, R, size, n = 16, 2, 32, 10
    inp = synth_inputs(UNetConfig(), size, size, f, seed=42)
    W = m._weights()
    d = DDIMScheduler()
    d.set_timesteps(n)
    ts, coef = d.timesteps.tolist(), d.coef_table()
    lat0 = inp["sample"][:1].float().to(dev)
    full = DenoiseEngine(W, size, size, f)
    _window(full, inp, dev)
    full.set_schedule(ts, coef, 3.5, guidance_rescale=0.7)
    ref = _run(full, lat0, 3)
    full.set_schedule(ts, coef, 3.5)
    plain = _run(full, lat0, 3)
    del full
    grp = ThreadGroup(R, monkeypatch)
    layout = shard_layout(R, f)

    def rank_fn(r):
        torch.cuda.set_device(dev)
        halves, frames = layout[r]
        eng = DenoiseEngine(W, size, size, f, Shard(halves=halves, frames=frames, group=grp, group_size=R,
                                                    rank_in_group=r, exchange="nccl"))
        _window(eng, inp, dev)
        eng.set_schedule(ts, coef, 3.5, guidance_rescale=0.7)
        out = _run(eng, lat0[:, :, list(frames)], 3)
        return out, eng._bufs[("rescale.totals", R, 4, torch.float64)].clone()

    res = grp.run(rank_fn)
    got = torch.cat([x for x, _ in res], dim=2)
    err, moved = rel_l2(got, ref), rel_l2(plain, ref)
    print(f"{R} thread-ranks vs unsharded, 3 DDIM steps at phi = 0.7: rel L2 = {err:.2e} (phi = 0 vs 0.7: "
          f"{moved:.2e}); totals bitwise equal on both ranks: {torch.equal(res[0][1], res[1][1])}")
    assert torch.equal(res[0][1], res[1][1])
    assert err < 5e-3 and moved > 5 * err


@pytest.mark.parametrize("exchange", ["peer", "nccl"])
def test_two_process_sharded_window_with_rescale(exchange):
    """tests/mgpu_rescale_worker.py under torchrun on two GPUs (skipped on fewer): a frame-sharded window at
    phi = 0.7 against the unsharded engine, eager and graph; every rank holds the same totals."""
    n = torch.cuda.device_count() if torch.cuda.is_available() else 0
    if n < 2:
        pytest.skip("needs >= 2 CUDA devices")
    port = 29541 if exchange == "peer" else 29542
    env = dict(os.environ, HALLO_B200_EXCHANGE=exchange, MASTER_ADDR="127.0.0.1", SIZE="32", FRAMES="16")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
                        "--master-addr", "127.0.0.1", "--master-port", str(port),
                        os.path.join(ROOT, "tests", "mgpu_rescale_worker.py")],
                       env=env, capture_output=True, text=True, timeout=900)
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("MGPU_RESULT ")]
    assert r.returncode == 0 and lines, r.stdout[-3000:] + r.stderr[-3000:]
    res = json.loads(lines[-1][len("MGPU_RESULT "):])
    print(res)
    assert all(c == 0 for c in res["device_errors_all_ranks"]), res
    assert res["totals_equal_eager"] and res["totals_equal_graph"], res
    assert res["eager_rel_l2"] < 5e-3 and res["graph_rel_l2"] < 5e-3, res


def test_face_animate_pipeline_guidance_rescale(model):
    """128x128, f = 4, 8 DDIM steps on the zero-terminal-SNR v-prediction schedule, CFG 3.5: guidance_rescale=0.0
    gives the video of a call without the keyword bitwise, through the same engine and graph; 0.7 changes it."""
    from hallo_b200.animate.face_animate import FaceAnimatePipeline
    from hallo_b200.scheduler import DDIMScheduler
    m, _ = model
    dev = _dev()
    H = W = 128
    f, n = 4, 8
    sched = DDIMScheduler(beta_start=0.00085, beta_end=0.012, beta_schedule="linear", clip_sample=False, steps_offset=1,
                          prediction_type="v_prediction", rescale_betas_zero_snr=True, timestep_spacing="trailing")
    pipe = FaceAnimatePipeline(vae=StubVAE(), reference_unet=StubReferenceNet(H // 8, W // 8), denoising_unet=m,
                               face_locator=StubFaceLocator((1,)), scheduler=sched, image_proj=StubProj((1, 4, 768)))
    pipe.to(device=dev, dtype=torch.float16)
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
    v_zero = call(guidance_rescale=0.0)
    assert m.engine(H // 8, W // 8, f) is eng and eng.graph is g                  # same engine, same graph
    v_r = call(guidance_rescale=0.7)
    assert eng.guidance_rescale == 0.7 and eng.graph is not g
    v_zero2 = call(guidance_rescale=0.0)
    e_r = rel_l2(v_r, v_default)
    print(f"pipeline, {n} DDIM steps: guidance_rescale=0.0 vs no keyword bitwise {torch.equal(v_zero, v_default)}; "
          f"0.7 vs no keyword {e_r:.2e}; 0.0 after 0.7 bitwise {torch.equal(v_zero2, v_default)}")
    assert torch.equal(v_zero, v_default) and torch.equal(v_zero2, v_default)
    assert torch.isfinite(v_r).all() and e_r > 1e-3 and tuple(v_r.shape) == (1, 3, f, H, W)
