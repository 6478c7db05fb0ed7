"""FaceAnimatePipeline -- the reference pipeline's call surface over the H100 denoising engine.

Mirrors hallo/animate/face_animate.py (FaceAnimatePipeline.__init__ :90-121, prepare_latents :136-188,
decode_latents :222-246, __call__ :249-442): same constructor modules, same __call__ keywords and tensor
contracts, same RNG contract (CPU generator -> initial latents), same output object (`.videos`, float32 CPU
(b, c, f, h, w) in [0, 1]).

What changed is who runs the 40-step loop (:384-427): instead of 40 x {torch.cat, UNet module walk, CFG,
scheduler.step} this hands the window to hallo_b200.engine.DenoiseEngine, which replays one captured CUDA
graph per step (UNet3D forward + CFG combine + DDIM update, all sm_90a kernels).  The VAE's encode / decode run on
hallo_b200.vae_engine (sm_90a kernels as well) when `vae` is an SD-1.5 AutoencoderKL on CUDA in fp16 / bf16, and
through the module itself otherwise.  ReferenceNet, face_locator and image_proj are the caller's modules.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Callable, List, Optional, Union

import numpy as np
import torch
import torch.nn.functional as F

from .. import vae_engine
from ..models.mutual_self_attention import ReferenceAttentionControl
from ..scheduler import coef_table_of


@dataclass
class FaceAnimatePipelineOutput:
    videos: Union[torch.Tensor, np.ndarray]


class FaceAnimatePipeline:
    def __init__(self, vae, reference_unet, denoising_unet, face_locator, image_proj, scheduler) -> None:
        self.vae = vae
        self.reference_unet = reference_unet
        self.denoising_unet = denoising_unet
        self.face_locator = face_locator
        self.image_proj = image_proj
        self.scheduler = scheduler
        self.vae_scale_factor: int = 2 ** (len(self.vae.config.block_out_channels) - 1)
        self.use_cuda_graph = True
        self.last_timing = {}
        self._vae_engine = None                  # (version key of self.vae, vae_engine.EngineVAE)

    def _vae_call(self):
        """What the VAE calls go through.  An nn.Module with the SD-1.5 AutoencoderKL grammar, on CUDA in fp16 or bf16,
        runs on the library's kernels (hallo_b200.vae_engine), packed once and repacked when its parameters change;
        anything else (another architecture, CPU, fp32) is called as it is."""
        m = self.vae
        if not vae_engine.runs_on_engine(m):
            return m
        key = vae_engine.version_key(m)
        if self._vae_engine is None or self._vae_engine[0] != key:
            self._vae_engine = None                                               # release the old packing first
            self._vae_engine = (key, vae_engine.EngineVAE(m))
        return self._vae_engine[1]

    # DiffusionPipeline.to(device=, dtype=) (scripts/inference.py:262)
    def to(self, device=None, dtype=None):
        for m in (self.vae, self.reference_unet, self.denoising_unet, self.face_locator, self.image_proj):
            if isinstance(m, torch.nn.Module):
                m.to(device=device, dtype=dtype)
        return self

    @property
    def device(self):
        return self.denoising_unet.device

    @property
    def _execution_device(self):
        return self.device

    def progress_bar(self, iterable=None, total=None):
        from tqdm import tqdm
        return tqdm(iterable, total=total) if iterable is not None else tqdm(total=total)

    def prepare_latents(self, batch_size, num_channels_latents, width, height, video_length, dtype, device,
                        generator=None, latents=None):
        """face_animate.py:136-188 + diffusers randn_tensor: a CPU generator draws on the CPU, then moves."""
        shape = (batch_size, num_channels_latents, video_length, height // self.vae_scale_factor,
                 width // self.vae_scale_factor)
        if isinstance(generator, list) and len(generator) != batch_size:
            raise ValueError(f"You have passed a list of generators of length {len(generator)}, but requested an "
                             f"effective batch size of {batch_size}.")
        if latents is None:
            gdev = generator.device if generator is not None and not isinstance(generator, list) else torch.device(device)
            latents = torch.randn(shape, generator=generator, device=gdev, dtype=dtype).to(device)
        else:
            latents = latents.to(device)
        return latents * self.scheduler.init_noise_sigma

    def decode_latents(self, latents, to_numpy: bool = True, chunk: int = 8):
        """face_animate.py:222-246: VAE decode of every frame, (x/2+0.5).clamp(0,1), float32.  The reference decodes
        one frame per call with a host sync each; the VAE is per-sample independent, so frames go through in chunks.
        to_numpy=True returns the reference's float32 numpy array on the CPU; False keeps the tensor on the device."""
        video_length = latents.shape[2]
        latents = 1 / 0.18215 * latents
        b = latents.shape[0]
        latents = latents.permute(0, 2, 1, 3, 4).reshape(b * video_length, *latents.shape[1:2], *latents.shape[3:])
        video = []
        vae = self._vae_call()
        for i in range(0, latents.shape[0], chunk):
            video.append(vae.decode(latents[i:i + chunk].to(self.vae.dtype)).sample)
        video = torch.cat(video)
        video = video.reshape(b, video_length, *video.shape[1:]).permute(0, 2, 1, 3, 4)
        video = (video / 2 + 0.5).clamp(0, 1).float()
        return video.cpu().numpy() if to_numpy else video

    def _preprocess_ref(self, x, height, width):
        """VaeImageProcessor.preprocess for tensor input: resize if needed, normalise only if data is in [0,1]."""
        if x.shape[-2:] != (height, width):
            x = F.interpolate(x, size=(height, width))
        if x.min() >= 0:
            x = 2.0 * x - 1.0
        return x

    @torch.no_grad()
    def prepare_static(self, face_emb, face_mask, pixel_values_full_mask, pixel_values_face_mask, pixel_values_lip_mask,
                       width, height, video_length, source_image=None):
        """Everything `__call__` derives from inputs that do not change from window to window of a clip
        (scripts/inference.py:285-339 passes the same face_emb / face_mask / masks / source image every iteration):
        image tokens (face_animate.py:291-298), the face-locator feature (:338-343, one frame, expanded), the CFG-doubled
        masks (:345-374) and the VAE latent of the source image (:330-336).  SURVEY.md 8f row 4: computed once per clip
        by hallo_b200.driver.ClipAnimator and handed back through `static=`; a plain `__call__` recomputes it."""
        unet = self.denoising_unet
        clip = face_emb.to(self.image_proj.device, self.image_proj.dtype)
        ehs = torch.cat([self.image_proj(torch.zeros_like(clip)), self.image_proj(clip)], dim=0)
        fm = face_mask.unsqueeze(1).to(dtype=self.face_locator.dtype, device=self.face_locator.device)   # (bs, 1, c, H, W)
        fm = fm.expand(fm.shape[0], video_length, *fm.shape[2:]).transpose(1, 2)       # (bs, c, f, H, W), stride 0 along f
        fm = self.face_locator(fm)
        mask_cond = torch.cat([torch.zeros_like(fm), fm], dim=0)

        def dup(ms):
            return [torch.cat([m] * 2).to(device=unet.device, dtype=unet.dtype) for m in ms]

        st = dict(ehs=ehs, mask_cond=mask_cond, full=dup(pixel_values_full_mask), face=dup(pixel_values_face_mask),
                  lip=dup(pixel_values_lip_mask), src_latent=None, src_key=None)
        if source_image is not None:
            src = self._preprocess_ref(source_image, height, width).to(dtype=self.vae.dtype, device=self.vae.device)
            st["src_latent"] = self._vae_call().encode(src).latent_dist.mean * 0.18215
        return st

    def _window_shard(self, video_length):
        """One process per GPU under torch.distributed: the window's frames are sharded over the ranks (hallo_b200.dist)."""
        try:
            import torch.distributed as dist
            if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
                from ..dist import plan_shard
                if getattr(self, "_shard", None) is None or self._shard[0] != video_length:
                    self._shard = (video_length, plan_shard(dist.get_rank(), dist.get_world_size(), video_length))
                return self._shard[1]
        except ImportError:
            pass
        return None

    @torch.no_grad()
    def __call__(self, ref_image, face_emb, audio_tensor, face_mask, pixel_values_full_mask, pixel_values_face_mask,
                 pixel_values_lip_mask, width, height, video_length, num_inference_steps, guidance_scale,
                 num_images_per_prompt=1, eta: float = 0.0, motion_scale: Optional[List[torch.Tensor]] = None,
                 generator=None, output_type: Optional[str] = "tensor", return_dict: bool = True,
                 callback: Optional[Callable[[int, int, torch.FloatTensor], None]] = None,
                 callback_steps: Optional[int] = 1, static: Optional[dict] = None, **kwargs):
        unet = self.denoising_unet
        device = self._execution_device
        height = height or unet.config.sample_size * self.vae_scale_factor
        width = width or unet.config.sample_size * self.vae_scale_factor
        do_cfg = guidance_scale > 1.0
        if not do_cfg:
            raise NotImplementedError("the engine implements the classifier-free-guidance path the reference ships")
        if eta != 0.0:
            raise NotImplementedError("eta != 0 (stochastic DDIM) is not part of the reference configuration")
        self.scheduler.set_timesteps(num_inference_steps, device=device)
        timesteps = self.scheduler.timesteps
        batch_size = 1
        e_a, e_b, e_c, e_d, e_e = (torch.cuda.Event(enable_timing=True) for _ in range(5))
        e_a.record()

        if static is None:
            static = self.prepare_static(face_emb, face_mask, pixel_values_full_mask, pixel_values_face_mask,
                                         pixel_values_lip_mask, width, height, video_length)
        ehs = static["ehs"]

        writer = ReferenceAttentionControl(self.reference_unet, do_classifier_free_guidance=do_cfg, mode="write",
                                           batch_size=batch_size, fusion_blocks="full")
        reader = ReferenceAttentionControl(unet, do_classifier_free_guidance=do_cfg, mode="read",
                                           batch_size=batch_size, fusion_blocks="full")

        latents = self.prepare_latents(batch_size * num_images_per_prompt, unet.in_channels, width, height,
                                       video_length, ehs.dtype, device, generator)

        ref = ref_image.reshape(-1, *ref_image.shape[2:])                       # "b f c h w -> (b f) c h w"
        if static.get("src_latent") is not None:                                # source latent hoisted: motion frames only
            mot = self._preprocess_ref(ref[1:], height, width).to(dtype=self.vae.dtype, device=self.vae.device)
            ref_latents = torch.cat([static["src_latent"], self._vae_call().encode(mot).latent_dist.mean * 0.18215], dim=0)
        else:
            ref = self._preprocess_ref(ref, height, width).to(dtype=self.vae.dtype, device=self.vae.device)
            ref_latents = self._vae_call().encode(ref).latent_dist.mean * 0.18215  # (1 + n_motion, 4, h, w)
        audio = torch.cat([torch.zeros_like(audio_tensor), audio_tensor], dim=0).to(dtype=unet.dtype, device=unet.device)
        e_b.record()

        # ReferenceNet once per window at t = 0 (face_animate.py:386-395)
        self.reference_unet(ref_latents.repeat(2, 1, 1, 1), torch.zeros_like(timesteps[0]),
                            encoder_hidden_states=ehs, return_dict=False)
        reader.update(writer)
        e_c.record()

        h8, w8 = height // self.vae_scale_factor, width // self.vae_scale_factor
        shard = self._window_shard(video_length)
        eng = unet.engine(h8, w8, video_length, shard)
        eng.begin_window(encoder_hidden_states=ehs, audio_embedding=audio, mask_cond_fea=static["mask_cond"],
                         full_mask=static["full"], face_mask=static["face"], lip_mask=static["lip"],
                         motion_scale=motion_scale, banks=unet._banks)
        eng.set_schedule(timesteps.tolist(), coef_table_of(self.scheduler), guidance_scale)
        frames = list(eng.shard.frames)
        eng.latents.copy_(latents[:, :, frames].float())
        if self.use_cuda_graph and callback is None and eng.graph is None:
            eng.capture()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i, t in enumerate(timesteps):
            eng.step()
            if callback is not None and i % callback_steps == 0:
                callback(i, t, eng.latents.to(latents.dtype))
        e1.record()
        local = eng.latents.to(latents.dtype)
        reader.clear()
        writer.clear()
        e_d.record()
        images = self.decode_latents(local, to_numpy=False)                     # (1, 3, fl, H, W) float32 in [0, 1], on device
        if shard is not None:
            import torch.distributed as dist
            parts = [torch.empty_like(images) for _ in range(shard.group_size)]
            dist.all_gather(parts, images.contiguous(), group=shard.group)     # frame groups in rank order
            images = torch.cat(parts, dim=2)
        e_e.record()
        self.last_device_video = images                                         # the driver takes motion frames from here
        self.last_events = dict(prep=(e_a, e_b), refnet=(e_b, e_c), window_setup=(e_c, e0), denoise=(e0, e1),
                                decode=(e_d, e_e))
        self.last_timing = {"steps": len(timesteps), "_events": True}
        if output_type == "tensor" or output_type == "device":
            out = images if output_type == "device" else images.cpu()
        else:
            out = images.cpu().numpy()
        if output_type != "device":
            self.last_timing["denoise_ms"] = e0.elapsed_time(e1)                # (the .cpu() above synchronised)
        if not return_dict:
            return out
        return FaceAnimatePipelineOutput(videos=out)

    def timing_ms(self) -> dict:
        """Per-phase device times of the last window (CUDA events; call after a synchronisation)."""
        return {k: a.elapsed_time(b) for k, (a, b) in self.last_events.items()}
