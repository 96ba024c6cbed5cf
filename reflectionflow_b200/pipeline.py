"""B200FluxPipeline — the diffusers FluxPipeline call surface the reference touches, over the
CUDA DiT:

  * `pipe(prompt=..|prompt_embeds=.., latents=.., guidance_scale=.., num_inference_steps=..,
          height=.., width=..).images`                       tts/tts_t2i_noise_scaling.py:60
  * `generate(pipe, conditions=[Condition], model_config=.., default_lora=True, **kwargs)`
                                                              train_flux/flux/generate.py:75-84
  * the attributes generate.py reads: check_inputs, encode_prompt, prepare_latents,
    _pack_latents/_unpack_latents/_prepare_latent_image_ids, scheduler, vae_scale_factor,
    set_progress_bar_config, load_lora_weights, to()      generate.py:114-131,148-174,193-213,302-310

Boundary (SURVEY.md §0.7, App. B): the reference draws seeds, init noise and condition latents
from unseeded global RNGs; here they are explicit inputs — `latents=`, `prompt_embeds=`,
`Condition(latents=...)` — so that a run is reproducible.  Text encoders (T5/CLIP) and the VAE are
the "next" tier (SURVEY.md §8f): until they are native, prompts must arrive as embeddings (or
through a user-supplied `text_encoder_hook`) and `output_type` must be "latent".
"""
from __future__ import annotations

import os
from contextlib import contextmanager
from dataclasses import dataclass
from typing import Any, Callable, Dict, List, Optional, Union

import numpy as np
import torch

from .config import FluxDiTConfig
from .scheduler import FlowMatchEulerDiscreteScheduler, calculate_shift
from .transformer import B200FluxTransformer2DModel, lora_scale

# train_flux/flux/condition.py:10-21.  The tts path uses "cot"; the DiT treats every type alike (the type-id column is
# produced but not consumed, transformer.py:133), so the other types only differ in how `raw_img` becomes the condition.
condition_dict = {"depth": 0, "canny": 1, "subject": 4, "coloring": 6, "deblurring": 7, "depth_pred": 8, "fill": 9,
                  "sr": 10, "cartoon": 11, "cot": 12}


@dataclass
class FluxPipelineOutput:
    images: Any


def flow_match_schedule(num_inference_steps: int, image_seq_len: int):
    """(timesteps fp32 [N], sigmas fp32 [N+1]) exactly as generate.py:193-209 builds them."""
    s = FlowMatchEulerDiscreteScheduler()
    sig = np.linspace(1.0, 1 / num_inference_steps, num_inference_steps)
    s.set_timesteps(sigmas=sig, mu=calculate_shift(image_seq_len))
    return s.timesteps, s.sigmas


class Condition:
    """train_flux/flux/condition.py:24-132 for the `cot` type: a parent image whose VAE latents
    join the sequence as condition tokens.  `latents` ([1, n, 64] packed, already shifted/scaled)
    may be given explicitly — the reference samples them from the VAE posterior with no
    generator (pipeline_tools.py:10), which is not reproducible.

    Image guidance (generate(..., image_guidance_scale != 1)) re-encodes the condition every step: the reference's
    `condition.encode(self, empty=True)` encodes the real image again (condition.py:121), a fresh posterior sample.
    With explicit `latents`, `uncond_latents` ([n_steps, *latents.shape]) gives those samples U_i; without it U_i =
    `latents`.  From an image, each U_i draws its posterior noise after the one of `latents`, from `generator` (else
    the global CPU RNG)."""

    def __init__(self, condition_type: str = "cot", raw_img=None, condition=None, mask=None,
                 position_delta=None, latents: Optional[torch.Tensor] = None,
                 eps: Optional[torch.Tensor] = None, generator: Optional[torch.Generator] = None,
                 uncond_latents: Optional[torch.Tensor] = None):
        if condition_type not in condition_dict:
            raise NotImplementedError(f"Condition type {condition_type} not implemented")
        assert mask is None, "Mask not supported yet"
        assert raw_img is not None or condition is not None or latents is not None
        self.condition_type = condition_type
        self.condition = condition
        if raw_img is not None:
            self.condition = self.get_condition(condition_type, raw_img)
        self.position_delta = position_delta
        self.latents = latents
        self.eps, self.generator = eps, generator  # posterior noise of the VAE encode (explicit)
        if uncond_latents is not None and latents is None:
            raise ValueError("uncond_latents go with explicit latents; a Condition from an image samples them")
        self.uncond_latents = uncond_latents

    def get_condition(self, condition_type: str, raw_img):
        """condition.py:43-80: raw image -> condition image.  "depth" needs the depth-anything network (not reachable
        offline); for "cot" / "sr" / "depth_pred" the reference has no rule (pass `condition=`): the image is taken as is."""
        if condition_type == "depth":
            raise NotImplementedError('"depth" conditions need the depth-estimation model (condition.py:49-59); '
                                      "pass the depth map as condition=")
        if condition_type == "canny":
            import cv2
            from PIL import Image
            return Image.fromarray(cv2.Canny(np.array(raw_img), 100, 200)).convert("RGB")
        if condition_type == "coloring":
            return raw_img.convert("L").convert("RGB")
        if condition_type == "deblurring":
            from PIL import ImageFilter
            return raw_img.convert("RGB").filter(ImageFilter.GaussianBlur(10)).convert("RGB")
        if condition_type in ("fill", "cartoon"):
            return raw_img.convert("RGB")
        return raw_img  # "subject" (:65-66) and the types without a rule

    @property
    def type_id(self) -> int:
        return condition_dict[self.condition_type]

    @classmethod
    def get_type_id(cls, condition_type: str) -> int:
        return condition_dict[condition_type]

    def encode(self, pipe: "B200FluxPipeline", empty: bool = False):
        if self.latents is not None:
            tokens = self.latents.to(pipe.device, pipe.dtype)
            side = int(round(tokens.shape[1] ** 0.5))
            ids = pipe._prepare_latent_image_ids(tokens.shape[0], side, side, pipe.device, pipe.dtype)
        else:
            tokens, ids = pipe.encode_images(self.condition, eps=self.eps, generator=self.generator)
        ids = ids.clone()
        if self.position_delta is None and self.condition_type == "subject" and self.condition is not None:
            self.position_delta = [0, -self.condition.size[0] // 16]  # condition.py:123-124
        if self.position_delta is not None:
            ids[:, 1] += self.position_delta[0]
            ids[:, 2] += self.position_delta[1]
        type_id = torch.ones_like(ids[:, :1]) * self.type_id
        return tokens, ids, type_id

    def encode_uncond(self, pipe: "B200FluxPipeline", n_steps: int) -> torch.Tensor:
        """The uncond condition tokens of an image-guided loop, [B, n_steps, n, 64]: row i is step i's
        `condition.encode(self, empty=True)[0]` (generate.py:251).  Call after `encode`."""
        if self.latents is not None:
            c0 = self.latents
            if self.uncond_latents is None:
                return c0[:, None].expand(c0.shape[0], n_steps, *c0.shape[1:])
            if tuple(self.uncond_latents.shape) != (n_steps,) + tuple(c0.shape):
                raise ValueError(f"uncond_latents has shape {tuple(self.uncond_latents.shape)}, expected "
                                 f"{(n_steps,) + tuple(c0.shape)} (steps, *latents.shape)")
            return self.uncond_latents.transpose(0, 1)
        return torch.stack([pipe.encode_images(self.condition, generator=self.generator)[0]
                            for _ in range(n_steps)], dim=1)


class B200FluxPipeline:
    vae_scale_factor = 8
    default_sample_size = 128
    _callback_tensor_inputs = ["latents", "prompt_embeds"]

    def __init__(self, transformer: B200FluxTransformer2DModel,
                 text_encoder_hook: Optional[Callable] = None, vae=None):
        self.transformer = transformer
        self.scheduler = FlowMatchEulerDiscreteScheduler()
        self.text_encoder_hook = text_encoder_hook  # (prompt, prompt_2, max_len) -> (embeds, pooled)
        self.vae = vae
        self.device = transformer.device
        self.dtype = torch.bfloat16
        self._execution_device = self.device
        self._guidance_scale = 3.5
        self._joint_attention_kwargs = None
        self._interrupt = False
        self._num_timesteps = 0
        self._progress = {}

    # ------------------------------------------------------------------ construction
    @classmethod
    def from_synthetic(cls, config=None, seed: int = 0, device="cuda:0", lora_rank: int = 0,
                       with_vae: bool = False):
        """Random-init FLUX.1-dev-shaped DiT (+ VAE decoder) — no checkpoints exist offline."""
        t = B200FluxTransformer2DModel(FluxDiTConfig.from_any(config or FluxDiTConfig()),
                                       lora_rank=lora_rank, device=device)
        t.init_synthetic_weights(seed)
        vae = None
        if with_vae:
            from .vae import B200AutoencoderKL
            vae = B200AutoencoderKL(device).init_synthetic_weights(seed + 1)
        return cls(t, vae=vae)

    @classmethod
    def from_state_dict(cls, state_dict, config=None, device="cuda:0", lora_rank: int = 0):
        t = B200FluxTransformer2DModel(FluxDiTConfig.from_any(config or FluxDiTConfig()),
                                       lora_rank=lora_rank, device=device)
        t.load_state_dict(state_dict)
        return cls(t)

    @classmethod
    def from_pretrained(cls, pretrained_model_name_or_path, cache_dir=None, torch_dtype=torch.bfloat16,
                        device="cuda:0", lora_rank: int = 0):
        """DiffusionPipeline.from_pretrained(name, torch_dtype=.., cache_dir=..) (tts_reflectionflow.py:498-502)
        for a FLUX.1-dev checkpoint in diffusers layout: a local directory, or a repo id already in the hub
        cache (`cache_dir`, default $HF_HUB_CACHE / $HF_HOME).  Nothing is downloaded.  Transformer, VAE, T5 /
        CLIP, their tokenizers and the scheduler all come from that directory; every config is checked before
        any device memory is allocated.  `lora_rank` sizes the adapter slots (checkpoint.max_lora_rank reads it
        from an adapter file); adapters load through load_lora_weights."""
        from . import checkpoint as ck
        from .text import B200TextEncoders
        from .vae import B200AutoencoderKL
        ck.check_dtype(torch_dtype)
        root = ck.resolve(pretrained_model_name_or_path, cache_dir)
        ck.check_model_index(root)
        join = lambda comp, name="config.json": os.path.join(root, comp, name)  # noqa: E731
        ck.dit_config(ck.read_json(join("transformer")))
        ck.vae_config(ck.read_json(join("vae")))
        ck.text_config(ck.read_json(join("text_encoder")), ck.read_json(join("text_encoder_2")))
        sched = ck.scheduler_config(ck.read_json(join("scheduler", "scheduler_config.json")))
        tokenizer, tokenizer_2 = ck.tokenizer_fns(root)
        transformer = B200FluxTransformer2DModel.from_pretrained(join("transformer", ""), lora_rank=lora_rank,
                                                                 device=device)
        vae = B200AutoencoderKL.from_pretrained(join("vae", ""), device=device)
        enc = B200TextEncoders.from_pretrained(join("text_encoder", ""), join("text_encoder_2", ""), device=device)
        pipe = cls(transformer, text_encoder_hook=enc.as_hook(tokenizer, tokenizer_2), vae=vae)
        pipe.scheduler = FlowMatchEulerDiscreteScheduler(**sched)
        pipe.text_encoders = enc
        return pipe

    def to(self, *a, **k):
        return self

    def set_progress_bar_config(self, **kw):
        self._progress.update(kw)

    def load_lora_weights(self, lora, adapter_name: str = "reflection", alpha: Optional[float] = None):
        """pipe.load_lora_weights(lora_path, adapter_name=...) (tts_reflectionflow.py:503-505):
        `lora` is a state dict / {module: (A, B)} mapping, a .safetensors path, or a directory holding
        pytorch_lora_weights.safetensors (what train_flux's save_lora writes, train/model.py:87-92)."""
        if isinstance(lora, (str, os.PathLike)):
            from safetensors.torch import load_file
            if os.path.isdir(lora):
                lora = os.path.join(lora, "pytorch_lora_weights.safetensors")
            lora = load_file(lora)
        self.transformer.load_lora(lora, alpha)

    def unload_lora_weights(self):
        """pipe.unload_lora_weights() (commented out at tts_reflectionflow.py:507): every LoRA target is unset."""
        self.transformer.unload_lora()

    def set_adapters(self, *a, **k):
        pass

    def maybe_free_model_hooks(self):
        pass

    @property
    def guidance_scale(self):
        return self._guidance_scale

    @property
    def joint_attention_kwargs(self):
        return self._joint_attention_kwargs

    @property
    def interrupt(self):
        return self._interrupt

    @property
    def num_timesteps(self):
        return self._num_timesteps

    @contextmanager
    def progress_bar(self, total=None):
        class _PB:
            def update(self_inner, n=1):
                pass
        yield _PB()

    # ------------------------------------------------------------------ diffusers helpers
    def check_inputs(self, prompt, prompt_2, height, width, prompt_embeds=None,
                     pooled_prompt_embeds=None, callback_on_step_end_tensor_inputs=None,
                     max_sequence_length=None):
        if height % (self.vae_scale_factor * 2) != 0 or width % (self.vae_scale_factor * 2) != 0:
            raise ValueError(f"`height` and `width` have to be divisible by {self.vae_scale_factor * 2} "
                             f"but are {height} and {width}.")
        if prompt is not None and prompt_embeds is not None:
            raise ValueError("Cannot forward both `prompt` and `prompt_embeds`. Please make sure to "
                             "only forward one of the two.")
        if prompt_2 is not None and prompt_embeds is not None:
            raise ValueError("Cannot forward both `prompt_2` and `prompt_embeds`.")
        if prompt is None and prompt_embeds is None:
            raise ValueError("Provide either `prompt` or `prompt_embeds`. Cannot leave both undefined.")
        if prompt is not None and not isinstance(prompt, (str, list)):
            raise ValueError(f"`prompt` has to be of type `str` or `list` but is {type(prompt)}")
        if prompt_embeds is not None and pooled_prompt_embeds is None:
            raise ValueError("If `prompt_embeds` are provided, `pooled_prompt_embeds` also have to be "
                             "passed.")
        if max_sequence_length is not None and max_sequence_length > 512:
            raise ValueError(f"`max_sequence_length` cannot be greater than 512 but is {max_sequence_length}")
        if callback_on_step_end_tensor_inputs is not None and not all(
                k in self._callback_tensor_inputs for k in callback_on_step_end_tensor_inputs):
            raise ValueError(f"`callback_on_step_end_tensor_inputs` has to be in {self._callback_tensor_inputs}, but "
                             f"found {[k for k in callback_on_step_end_tensor_inputs if k not in self._callback_tensor_inputs]}")

    def encode_prompt(self, prompt=None, prompt_2=None, device=None, num_images_per_prompt: int = 1,
                      prompt_embeds=None, pooled_prompt_embeds=None, max_sequence_length: int = 512,
                      lora_scale=None):
        device = device or self.device
        if prompt_embeds is None:
            if self.text_encoder_hook is None:
                raise NotImplementedError(
                    "no text encoders are attached (T5/CLIP are the next tier, SURVEY.md §8f): pass "
                    "prompt_embeds/pooled_prompt_embeds or construct the pipeline with text_encoder_hook")
            prompt = [prompt] if isinstance(prompt, str) else prompt
            prompt_2 = prompt_2 or prompt
            prompt_2 = [prompt_2] if isinstance(prompt_2, str) else prompt_2
            prompt_embeds, pooled_prompt_embeds = self.text_encoder_hook(prompt, prompt_2,
                                                                         max_sequence_length)
        prompt_embeds = prompt_embeds.to(device=device, dtype=self.dtype)
        pooled_prompt_embeds = pooled_prompt_embeds.to(device=device, dtype=self.dtype)
        if num_images_per_prompt != 1:
            prompt_embeds = prompt_embeds.repeat_interleave(num_images_per_prompt, dim=0)
            pooled_prompt_embeds = pooled_prompt_embeds.repeat_interleave(num_images_per_prompt, dim=0)
        text_ids = torch.zeros(prompt_embeds.shape[1], 3, device=device, dtype=self.dtype)
        return prompt_embeds, pooled_prompt_embeds, text_ids

    @staticmethod
    def _pack_latents(latents, batch_size, num_channels_latents, height, width):
        latents = latents.view(batch_size, num_channels_latents, height // 2, 2, width // 2, 2)
        latents = latents.permute(0, 2, 4, 1, 3, 5)
        return latents.reshape(batch_size, (height // 2) * (width // 2), num_channels_latents * 4)

    @staticmethod
    def _unpack_latents(latents, height, width, vae_scale_factor):
        batch_size, num_patches, channels = latents.shape
        height = 2 * (int(height) // (vae_scale_factor * 2))
        width = 2 * (int(width) // (vae_scale_factor * 2))
        latents = latents.view(batch_size, height // 2, width // 2, channels // 4, 2, 2)
        latents = latents.permute(0, 3, 1, 4, 2, 5)
        return latents.reshape(batch_size, channels // (2 * 2), height, width)

    @staticmethod
    def _prepare_latent_image_ids(batch_size, height, width, device, dtype):
        ids = torch.zeros(height, width, 3)
        ids[..., 1] = ids[..., 1] + torch.arange(height)[:, None]
        ids[..., 2] = ids[..., 2] + torch.arange(width)[None, :]
        return ids.reshape(height * width, 3).to(device=device, dtype=dtype)

    def prepare_latents(self, batch_size, num_channels_latents, height, width, dtype, device,
                        generator, latents=None):
        height = 2 * (int(height) // (self.vae_scale_factor * 2))
        width = 2 * (int(width) // (self.vae_scale_factor * 2))
        ids = self._prepare_latent_image_ids(batch_size, height // 2, width // 2, device, dtype)
        if latents is not None:
            return latents.to(device=device, dtype=dtype), ids
        shape = (batch_size, num_channels_latents, height, width)
        if isinstance(generator, list) and len(generator) != batch_size:
            raise ValueError("generator list length must match batch size")
        # diffusers randn_tensor: a CPU generator draws on the CPU (in dtype), then moves
        gdev = "cpu" if generator is None or getattr(generator, "device", torch.device("cpu")).type == "cpu" else device
        noise = torch.randn(shape, generator=generator, device=gdev, dtype=dtype).to(device)
        return self._pack_latents(noise, batch_size, num_channels_latents, height, width), ids

    def encode_images(self, images, eps: Optional[torch.Tensor] = None,
                      generator: Optional[torch.Generator] = None):
        """train_flux/flux/pipeline_tools.py:7-30: preprocess -> vae.encode -> posterior sample ->
        (z - shift) * scale -> pack, + position ids.  `images`: PIL image(s) or uint8 [B, H, W, 3]
        (sizes must be multiples of 16).  The posterior noise is `eps` (bf16 [16, H/8, W/8]) or drawn
        from `generator`; with neither it comes from the global CPU RNG (the reference samples it
        with no generator at all, App. B.4)."""
        if self.vae is None:
            raise NotImplementedError("no VAE attached: construct Condition(latents=...) or build the "
                                      "pipeline with vae=B200AutoencoderKL(...)")
        if not torch.is_tensor(images):
            imgs = images if isinstance(images, (list, tuple)) else [images]
            images = torch.stack([torch.from_numpy(np.array(im.convert("RGB"))) for im in imgs])
        if images.dim() == 3:
            images = images[None]
        B, H, W, _ = images.shape
        if H % 16 or W % 16:
            raise ValueError("condition image sides must be multiples of 16")
        if eps is None:
            eps = torch.randn((16, H // 8, W // 8), generator=generator, dtype=self.dtype)
        tokens = self.vae.encode_packed(images, eps)
        ids = self._prepare_latent_image_ids(B, H // 16, W // 16, self.device, self.dtype)
        return tokens, ids

    # ------------------------------------------------------------------ the denoise call
    def _denoise(self, latents, prompt_embeds, pooled, text_ids, image_ids, num_inference_steps,
                 guidance_scale, timesteps=None, condition_latents=None, condition_ids=None,
                 model_config=None, condition_scale: float = 1.0, image_guidance_scale: float = 1.0,
                 uncond_latents=None, callback_on_step_end=None, callback_on_step_end_tensor_inputs=("latents",)):
        if timesteps is not None:
            raise NotImplementedError("custom `timesteps` are not supported (the reference passes sigmas)")
        sigmas = np.linspace(1.0, 1 / num_inference_steps, num_inference_steps)
        mu = calculate_shift(latents.shape[1], self.scheduler.config.base_image_seq_len,
                             self.scheduler.config.max_image_seq_len, self.scheduler.config.base_shift,
                             self.scheduler.config.max_shift)
        self.scheduler.set_timesteps(sigmas=sigmas, mu=mu, device="cpu")
        ts = self.scheduler.timesteps
        self._num_timesteps = len(ts)
        # generate.py:222,240: t -> latents dtype (bf16), then / 1000 in bf16
        t_in = ts.to(self.dtype) / 1000
        hook = None
        if callback_on_step_end is not None:
            hook = self._step_hook(callback_on_step_end, callback_on_step_end_tensor_inputs, ts)
        return self.transformer.denoise(latents, prompt_embeds, pooled, t_in, self.scheduler.sigmas,
                                        guidance_scale, image_ids, text_ids, condition_latents,
                                        condition_ids, model_config, condition_scale,
                                        **({} if image_guidance_scale == 1.0 else dict(
                                            image_guidance_scale=image_guidance_scale,
                                            uncond_condition_latents=uncond_latents)),
                                        **({} if hook is None else dict(step_hook=hook)))

    def _step_hook(self, callback, tensor_inputs, timesteps):
        """generate.py:283-290 as a step hook of `transformer.denoise`: after step i, `callback(self, i, t,
        callback_kwargs)` with t = scheduler.timesteps[i] (0-d fp32 on the device) and the tensors named by
        `tensor_inputs`; its "latents" / "prompt_embeds" feed the next step, or are the result of the call (other keys
        are ignored, as the reference's `pop`).  Once the callback sets `self._interrupt`, no further step runs
        (generate.py:218-219), and the latents it returned in that step are the result."""
        ts = timesteps.to(self.device)

        def hook(i, latents, prompt_embeds):
            tensors = {"latents": latents, "prompt_embeds": prompt_embeds}
            out = callback(self, i, ts[i], {k: tensors[k] for k in tensor_inputs})
            return out.pop("latents", latents), out.pop("prompt_embeds", prompt_embeds), self.interrupt
        return hook

    def _finish(self, latents, height, width, output_type, return_dict):
        if output_type == "latent":
            image = latents
        else:
            if self.vae is None:
                raise NotImplementedError(
                    "no VAE attached: call with output_type='latent' or construct the pipeline with "
                    "vae=B200AutoencoderKL(...)")
            # generate.py:302-307 in one device call: unpack, / scaling + shift, decode, postprocess
            if output_type == "pil":
                from .vae import to_pil
                image = to_pil(self.vae.decode_packed(latents, height, width, "u8"))
            elif output_type == "np":
                image = self.vae.decode_packed(latents, height, width, "u8").cpu().numpy().astype("float32") / 255.0
            elif output_type == "pt":
                image = self.vae.decode_packed(latents, height, width, "pt")
            elif output_type == "u8":  # extension: uint8 [B, H, W, 3] left on the device
                image = self.vae.decode_packed(latents, height, width, "u8")
            else:
                raise ValueError(f"output_type {output_type!r} not supported")
        if not return_dict:
            return (image,)
        return FluxPipelineOutput(images=image)

    @torch.no_grad()
    def __call__(self, prompt: Union[str, List[str]] = None, prompt_2=None, height: Optional[int] = None,
                 width: Optional[int] = None, num_inference_steps: int = 28, timesteps=None,
                 guidance_scale: float = 3.5, num_images_per_prompt: int = 1, generator=None,
                 latents: Optional[torch.Tensor] = None, prompt_embeds=None,
                 pooled_prompt_embeds=None, output_type: str = "pil", return_dict: bool = True,
                 joint_attention_kwargs: Optional[Dict[str, Any]] = None,
                 callback_on_step_end=None, callback_on_step_end_tensor_inputs=("latents",),
                 max_sequence_length: int = 512, **_):
        """diffusers FluxPipeline.__call__ (entry A)."""
        height = height or self.default_sample_size * self.vae_scale_factor
        width = width or self.default_sample_size * self.vae_scale_factor
        self.check_inputs(prompt, prompt_2, height, width, prompt_embeds=prompt_embeds,
                          pooled_prompt_embeds=pooled_prompt_embeds,
                          callback_on_step_end_tensor_inputs=callback_on_step_end_tensor_inputs,
                          max_sequence_length=max_sequence_length)
        self._guidance_scale = guidance_scale
        self._joint_attention_kwargs = joint_attention_kwargs
        self._interrupt = False
        if prompt is not None and isinstance(prompt, str):
            batch_size = 1
        elif prompt is not None and isinstance(prompt, list):
            batch_size = len(prompt)
        else:
            batch_size = prompt_embeds.shape[0]
        device = self._execution_device
        prompt_embeds, pooled_prompt_embeds, text_ids = self.encode_prompt(
            prompt=prompt, prompt_2=prompt_2, prompt_embeds=prompt_embeds,
            pooled_prompt_embeds=pooled_prompt_embeds, device=device,
            num_images_per_prompt=num_images_per_prompt, max_sequence_length=max_sequence_length)
        num_channels_latents = self.transformer.config.in_channels // 4
        latents, latent_image_ids = self.prepare_latents(
            batch_size * num_images_per_prompt, num_channels_latents, height, width,
            prompt_embeds.dtype, device, generator, latents)
        latents = self._denoise(latents, prompt_embeds, pooled_prompt_embeds, text_ids,
                                latent_image_ids, num_inference_steps, guidance_scale, timesteps,
                                callback_on_step_end=callback_on_step_end,
                                callback_on_step_end_tensor_inputs=callback_on_step_end_tensor_inputs)
        return self._finish(latents, height, width, output_type, return_dict)


def encode_images(pipeline: "B200FluxPipeline", images, eps: Optional[torch.Tensor] = None,
                  generator: Optional[torch.Generator] = None):
    """Module-level form of train_flux/flux/pipeline_tools.py:7-30 (`encode_images(pipeline, images)`):
    -> (image tokens [B, (H/16)(W/16), 64], position ids).  The posterior noise is explicit (see the method)."""
    return pipeline.encode_images(images, eps=eps, generator=generator)


def prepare_text_input(pipeline: "B200FluxPipeline", prompts, max_sequence_length: int = 512, prompts_2=None):
    """train_flux/flux/pipeline_tools.py:33-52: `encode_prompt` with the reference's fixed arguments
    -> (prompt_embeds, pooled_prompt_embeds, text_ids)."""
    return pipeline.encode_prompt(prompt=prompts, prompt_2=prompts_2, prompt_embeds=None,
                                  pooled_prompt_embeds=None, device=pipeline.device, num_images_per_prompt=1,
                                  max_sequence_length=max_sequence_length, lora_scale=None)


def get_config(config_path: str = None) -> dict:
    """train_flux/flux/generate.py:16-22: the yaml named by `config_path`, else by $XFL_CONFIG, else {}."""
    import os
    config_path = config_path or os.environ.get("XFL_CONFIG")
    if not config_path:
        return {}
    import yaml
    with open(config_path, "r") as f:
        return yaml.safe_load(f) or {}


def seed_everything(seed: int = 42):
    """train_flux/flux/generate.py:68-72 (the cudnn flag has no meaning here: no cuDNN on the path)."""
    import numpy as np
    torch.manual_seed(seed)
    np.random.seed(seed)


@torch.no_grad()
def generate(pipeline: B200FluxPipeline, conditions: List[Condition] = None, config_path: str = None,
             model_config: Optional[Dict[str, Any]] = {}, condition_scale: float = 1.0,
             default_lora: bool = False, image_guidance_scale: float = 1.0, **params):
    """train_flux/flux/generate.py:75-321 (entry B): FluxPipeline.__call__ + one condition stream.
    Same keyword surface (prepare_params, generate.py:25-65); defaults 512x512 / 28 steps / 3.5."""
    model_config = model_config or get_config(config_path).get("model", {}) or {}
    self = pipeline
    guided = image_guidance_scale != 1.0  # generate.py:250-272
    if guided and conditions is None:  # a NameError upstream (`condition` is unbound)
        raise ValueError("image_guidance_scale != 1 guides over the condition stream: pass a condition")
    if guided and not self.transformer.config.guidance_embeds:  # a TypeError upstream (ones_like(None))
        raise ValueError("image_guidance_scale != 1 runs its uncond branch at guidance 1: it needs a model with "
                         "guidance_embeds=True")
    prompt = params.get("prompt")
    prompt_2 = params.get("prompt_2")
    height = params.get("height", 512) or self.default_sample_size * self.vae_scale_factor
    width = params.get("width", 512) or self.default_sample_size * self.vae_scale_factor
    num_inference_steps = params.get("num_inference_steps", 28)
    guidance_scale = params.get("guidance_scale", 3.5)
    num_images_per_prompt = params.get("num_images_per_prompt", 1)
    prompt_embeds = params.get("prompt_embeds")
    pooled_prompt_embeds = params.get("pooled_prompt_embeds")
    max_sequence_length = params.get("max_sequence_length", 512)
    callback_on_step_end_tensor_inputs = params.get("callback_on_step_end_tensor_inputs", ["latents"])
    self.check_inputs(prompt, prompt_2, height, width, prompt_embeds=prompt_embeds,
                      pooled_prompt_embeds=pooled_prompt_embeds,
                      callback_on_step_end_tensor_inputs=callback_on_step_end_tensor_inputs,
                      max_sequence_length=max_sequence_length)
    self._guidance_scale = guidance_scale
    self._joint_attention_kwargs = params.get("joint_attention_kwargs")
    self._interrupt = False
    if prompt is not None and isinstance(prompt, str):
        batch_size = 1
    elif prompt is not None and isinstance(prompt, list):
        batch_size = len(prompt)
    else:
        batch_size = prompt_embeds.shape[0]
    device = self._execution_device
    prompt_embeds, pooled_prompt_embeds, text_ids = self.encode_prompt(
        prompt=prompt, prompt_2=prompt_2, prompt_embeds=prompt_embeds,
        pooled_prompt_embeds=pooled_prompt_embeds, device=device,
        num_images_per_prompt=num_images_per_prompt, max_sequence_length=max_sequence_length)
    latents, latent_image_ids = self.prepare_latents(
        batch_size * num_images_per_prompt, self.transformer.config.in_channels // 4, height, width,
        prompt_embeds.dtype, device, params.get("generator"), params.get("latents"))
    cond_lat = cond_ids = None
    if conditions is not None:  # generate.py:178 `conditions is not None or []`
        assert len(conditions) <= 1, "Only one condition is supported for now."
        if len(conditions) == 0:
            raise RuntimeError("conditions=[] fails upstream too (torch.cat of an empty list, "
                               "SURVEY App. B.2): pass None or one Condition")
        if not default_lora:
            pipeline.set_adapters(conditions[0].condition_type)
        toks, ids = [], []
        for c in conditions:
            t, i, _type_id = c.encode(self)
            toks.append(t)
            ids.append(i)
        cond_lat = torch.cat(toks, dim=1)
        cond_ids = torch.cat(ids, dim=0)
    unc_lat = conditions[-1].encode_uncond(self, num_inference_steps) if guided else None
    # joint_attention_kwargs["scale"] reaches every step of the loop (generate.py:246 -> transformer.py:73-81)
    with lora_scale(self.transformer, self._joint_attention_kwargs):
        latents = self._denoise(latents, prompt_embeds, pooled_prompt_embeds, text_ids, latent_image_ids,
                                num_inference_steps, guidance_scale, params.get("timesteps"), cond_lat,
                                cond_ids, model_config, condition_scale, image_guidance_scale, unc_lat,
                                params.get("callback_on_step_end"), callback_on_step_end_tensor_inputs)
    return self._finish(latents, height, width, params.get("output_type", "pil"),
                        params.get("return_dict", True))
