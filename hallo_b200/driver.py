"""Clip driver: the sliding-window loop of scripts/inference.py:262-347 over hallo_b200's pipeline (SURVEY.md 8f rows
2-4).

The reference walks a clip in 16-frame windows; window t's reference stack is [source image, last n_motion frames of
window t-1] (the source image repeated for t = 0), its audio tokens are AudioProjModel(audio_emb[16t:16t+16]), and
windows are strictly sequential (motion-frame dependency).  What this driver changes, with identical results:
  * conditioning that is the same for every window is computed ONCE per clip (`FaceAnimatePipeline.prepare_static`:
    image tokens, face-locator feature, CFG-doubled masks, the source image's VAE latent) and the audio projection of
    ALL windows is one batched call (scripts/inference.py:314-320 runs it per window);
  * the decoded window stays on the device: the motion frames are taken from it there (the reference round-trips the
    whole window through host memory, inference.py:303-310) and finished windows are copied to the host asynchronously;
  * under torch.distributed each window is frame-sharded over the ranks (hallo_b200.dist); every rank runs the (small)
    ReferenceNet redundantly and decodes its own frames, the window's frames are all-gathered for the hand-off.
"""
from __future__ import annotations

import math
from typing import List, Optional, Sequence, Tuple

import torch

from .engine import check_guidance_interval, check_guidance_rescale


def process_audio_emb(audio_emb: torch.Tensor) -> torch.Tensor:
    """scripts/inference.py:95-114: frame i gets the embeddings of frames i-2..i+2 (indices clamped to the clip):
    (S, 12, 768) -> (S, 5, 12, 768)."""
    S = audio_emb.shape[0]
    idx = (torch.arange(S).unsqueeze(1) + torch.arange(-2, 3).unsqueeze(0)).clamp_(0, S - 1)
    return audio_emb[idx]


def padded_sequence_length(seq_len: int, clip_length: int) -> int:
    """hallo/datasets/audio_processor.py:108-115: the audio is zero-padded to a whole number of windows."""
    if clip_length > 0 and seq_len % clip_length != 0:
        seq_len += clip_length - seq_len % clip_length
    return seq_len


def audio_frames(n_samples: int, sample_rate: int = 16000, fps: int = 25) -> int:
    """audio_processor.py:103: seq_len = ceil(samples / sample_rate * fps)  (30 s -> 750 frames -> 47 windows)."""
    return math.ceil(n_samples / sample_rate * fps)


def window_reference_stack(source_image: torch.Tensor, previous_window: Optional[torch.Tensor], n_motion_frames: int):
    """scripts/inference.py:292-312.  source_image (1, 3, H, W) in [-1, 1]; previous_window: the last pipeline output
    (1, 3, f, H, W) in [0, 1] or None.  -> (1, 1 + n_motion, 3, H, W)."""
    if previous_window is None:
        motion = source_image.repeat(n_motion_frames, 1, 1, 1)
    else:
        motion = previous_window[0].permute(1, 0, 2, 3)[-n_motion_frames:] * 2.0 - 1.0
        motion = motion.to(dtype=source_image.dtype, device=source_image.device)
    return torch.cat([source_image, motion], dim=0).unsqueeze(0)


class ClipAnimator:
    def __init__(self, pipeline, audio_proj, clip_length: int = 16, n_motion_frames: int = 2):
        self.pipeline, self.audio_proj = pipeline, audio_proj
        self.clip_length, self.n_motion_frames = clip_length, n_motion_frames
        self.window_timings: List[dict] = []

    @torch.no_grad()
    def __call__(self, source_image_pixels, source_image_face_region, source_image_face_emb, source_image_full_mask,
                 source_image_face_mask, source_image_lip_mask, audio_emb, audio_length: Optional[int] = None,
                 width: int = 512, height: int = 512, num_inference_steps: int = 40, guidance_scale: float = 3.5,
                 motion_scale: Sequence[float] = (1.0, 1.0, 1.0), generator=None, max_windows: Optional[int] = None,
                 hoist: bool = True, audio_guidance_scale: Optional[float] = None,
                 guidance_rescale: float = 0.0,
                 guidance_interval: Optional[Tuple[float, float]] = None) -> torch.Tensor:
        """Arguments as scripts/inference.py prepares them: source_image_pixels (3, H, W) in [-1, 1], face region
        (3, H, W), face embedding (512,), three lists of 4 masks (1, L_l), audio_emb (S, 5, 12, 768) already through
        process_audio_emb, S a multiple of clip_length.  Returns the clip (3, audio_length, H, W) float32 on the host.
        audio_guidance_scale: a separate guidance weight for the audio (FaceAnimatePipeline.__call__); None keeps the
        single guidance_scale.  guidance_rescale: phi in [0, 1] of guidance rescale (FaceAnimatePipeline.__call__),
        checked before any work; 0.0 leaves the guided prediction as it is.  guidance_interval: (t_lo, t_hi) in the
        scheduler's timestep units; steps outside it run unguided on the cond branch alone
        (FaceAnimatePipeline.__call__), checked before any work; None guides every step."""
        guidance_rescale = check_guidance_rescale(guidance_rescale)
        guidance_interval = check_guidance_interval(guidance_interval)
        pipe, cl = self.pipeline, self.clip_length
        dev = pipe.device
        src = source_image_pixels.unsqueeze(0).to(dev)
        face_region = source_image_face_region.unsqueeze(0)
        face_emb = torch.as_tensor(source_image_face_emb).reshape(1, -1)
        full_m = [m.repeat(cl, 1) for m in source_image_full_mask]
        face_m = [m.repeat(cl, 1) for m in source_image_face_mask]
        lip_m = [m.repeat(cl, 1) for m in source_image_lip_mask]
        times = audio_emb.shape[0] // cl
        if max_windows is not None:
            times = min(times, max_windows)
        generator = torch.manual_seed(42) if generator is None else generator     # inference.py:289
        static = None
        if hoist:
            static = pipe.prepare_static(face_emb, face_region, full_m, face_m, lip_m, width, height, cl, source_image=src)
            # all windows' audio tokens in one call (per-row independent: identical to the per-window calls)
            a = audio_emb[:times * cl].to(device=self.audio_proj.device, dtype=self.audio_proj.dtype)
            audio_tokens = self.audio_proj(a.unsqueeze(0))[0]                      # (times*cl, 32, 768)
        host_windows: List[torch.Tensor] = []
        copy_stream = torch.cuda.Stream(device=dev)
        previous = None
        self.window_timings = []
        for t in range(times):
            ref_stack = window_reference_stack(src, previous, self.n_motion_frames)
            if hoist:
                audio_tensor = audio_tokens[t * cl:(t + 1) * cl].unsqueeze(0)
            else:
                a = audio_emb[t * cl:(t + 1) * cl].unsqueeze(0).to(device=self.audio_proj.device, dtype=self.audio_proj.dtype)
                audio_tensor = self.audio_proj(a)
            out = pipe(ref_image=ref_stack, audio_tensor=audio_tensor, face_emb=face_emb, face_mask=face_region,
                       pixel_values_full_mask=full_m, pixel_values_face_mask=face_m, pixel_values_lip_mask=lip_m,
                       width=width, height=height, video_length=cl, num_inference_steps=num_inference_steps,
                       guidance_scale=guidance_scale, generator=generator, motion_scale=list(motion_scale),
                       static=static, output_type="device", audio_guidance_scale=audio_guidance_scale,
                       guidance_rescale=guidance_rescale, guidance_interval=guidance_interval)
            previous = out.videos                                                  # (1, 3, cl, H, W) on the device
            done = torch.cuda.Event()
            done.record()
            host = torch.empty(previous.shape, dtype=torch.float32, pin_memory=True)
            with torch.cuda.stream(copy_stream):                                   # D2H of window t overlaps window t+1
                copy_stream.wait_event(done)
                host.copy_(previous, non_blocking=True)
            previous.record_stream(copy_stream)
            host_windows.append(host)
            self.window_timings.append(dict(events=pipe.last_events))
        copy_stream.synchronize()
        torch.cuda.synchronize()
        for wt in self.window_timings:
            ev = wt.pop("events")
            wt.update({k: a.elapsed_time(b) for k, (a, b) in ev.items()})
        video = torch.cat(host_windows, dim=2).squeeze(0)                          # (3, times*cl, H, W)
        if audio_length is not None:
            video = video[:, :audio_length]
        return video
