"""B200AutoencoderKL — the FLUX VAE decoder on the device (rf_vae_* in include/rf_b200.h).

Replaces, for the pipeline tail at train_flux/flux/generate.py:302-307,
    latents = pipe._unpack_latents(latents, h, w, 8)
    latents = latents / vae.config.scaling_factor + vae.config.shift_factor
    image = vae.decode(latents, return_dict=False)[0]
    image = image_processor.postprocess(image, output_type="pil")
with one C-ABI call: packed latents in, uint8 HWC (or a bf16 CHW tensor) out."""
from __future__ import annotations

import ctypes
from typing import Dict, List, Optional

import torch

from . import _lib as L


class _Cfg(dict):
    __getattr__ = dict.__getitem__


class B200AutoencoderKL:
    def __init__(self, device="cuda:0", scaling_factor: float = 0.3611, shift_factor: float = 0.1159):
        if not torch.cuda.is_available():
            raise L.RFError("B200AutoencoderKL needs a CUDA device; there is no CPU fallback")
        self.device = torch.device(device)
        self.dtype = torch.bfloat16
        self.config = _Cfg(scaling_factor=scaling_factor, shift_factor=shift_factor, latent_channels=16,
                           block_out_channels=(128, 256, 512, 512))
        self._lib = L.load()
        self._h = ctypes.c_void_p()
        with torch.cuda.device(self.device):
            L.check(self._lib.rf_vae_create(ctypes.byref(self._h)), "rf_vae_create")

    def close(self):
        if getattr(self, "_h", None) and self._h.value:
            self._lib.rf_vae_destroy(self._h)
            self._h = ctypes.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @classmethod
    def from_pretrained(cls, vae_dir: str, device="cuda:0"):
        """A diffusers `vae/` directory: scaling / shift factors from its config.json (any other shape than the
        FLUX VAE's is refused before the handle is created), weights streamed from its safetensors (the FLUX
        VAE ships in fp32; they are cast to bf16 on the host)."""
        import os
        from . import checkpoint as ck
        factors = ck.vae_config(ck.read_json(os.path.join(vae_dir, "config.json")))
        stream = ck.SafetensorsStream(vae_dir, ck.vae_key)
        return cls(device, **factors).load_state_dict(stream)

    def load_state_dict(self, sd: Dict[str, torch.Tensor], strict: bool = True):
        """diffusers AutoencoderKL keys (`decoder.*` and `encoder.*`)."""
        with torch.cuda.device(self.device):
            for k, v in sd.items():
                if not (k.startswith("decoder.") or k.startswith("encoder.")):
                    continue
                t = v.detach().to(self.device, torch.bfloat16).contiguous()
                L.check(self._lib.rf_vae_load_weight(self._h, k.encode(), L.ptr(t), t.numel()),
                        f"rf_vae_load_weight({k})")
            if strict and self._lib.rf_vae_missing_weights(self._h) != 0:
                L.check(-4, "B200AutoencoderKL.load_state_dict (missing weights)")
        return self

    def init_synthetic_weights(self, seed: int = 0):
        """random-init decoder of the FLUX VAE architecture (no checkpoint exists offline)"""
        g = torch.Generator(device=self.device).manual_seed(seed)

        def put(key, t):
            t = t.to(torch.bfloat16).contiguous()
            L.check(self._lib.rf_vae_load_weight(self._h, key.encode(), L.ptr(t), t.numel()), key)

        def conv(key, cout, cin, k):
            put(key + ".weight", torch.randn(cout, cin, k, k, generator=g, device=self.device) / (cin * k * k) ** 0.5)
            put(key + ".bias", 0.05 * torch.randn(cout, generator=g, device=self.device))

        def norm(key, c):
            put(key + ".weight", 1 + 0.1 * torch.randn(c, generator=g, device=self.device))
            put(key + ".bias", 0.05 * torch.randn(c, generator=g, device=self.device))

        def resnet(key, cin, cout):
            norm(key + ".norm1", cin); conv(key + ".conv1", cout, cin, 3)
            norm(key + ".norm2", cout); conv(key + ".conv2", cout, cout, 3)
            if cin != cout:
                conv(key + ".conv_shortcut", cout, cin, 1)

        with torch.cuda.device(self.device):
            conv("decoder.conv_in", 512, 16, 3)
            resnet("decoder.mid_block.resnets.0", 512, 512)
            resnet("decoder.mid_block.resnets.1", 512, 512)
            a = "decoder.mid_block.attentions.0."
            norm(a + "group_norm", 512)
            for n in ("to_q", "to_k", "to_v", "to_out.0"):
                put(a + n + ".weight", torch.randn(512, 512, generator=g, device=self.device) / 512 ** 0.5)
                put(a + n + ".bias", 0.05 * torch.randn(512, generator=g, device=self.device))
            prev = 512
            for i, c in enumerate((512, 512, 256, 128)):
                for j in range(3):
                    resnet(f"decoder.up_blocks.{i}.resnets.{j}", prev if j == 0 else c, c)
                if i < 3:
                    conv(f"decoder.up_blocks.{i}.upsamplers.0.conv", c, c, 3)
                prev = c
            norm("decoder.conv_norm_out", 128)
            conv("decoder.conv_out", 3, 128, 3)
            conv("encoder.conv_in", 128, 3, 3)
            prev = 128
            for i, c in enumerate((128, 256, 512, 512)):
                for j in range(2):
                    resnet(f"encoder.down_blocks.{i}.resnets.{j}", prev if j == 0 else c, c)
                if i < 3:
                    conv(f"encoder.down_blocks.{i}.downsamplers.0.conv", c, c, 3)
                prev = c
            resnet("encoder.mid_block.resnets.0", 512, 512)
            resnet("encoder.mid_block.resnets.1", 512, 512)
            a = "encoder.mid_block.attentions.0."
            norm(a + "group_norm", 512)
            for n in ("to_q", "to_k", "to_v", "to_out.0"):
                put(a + n + ".weight", torch.randn(512, 512, generator=g, device=self.device) / 512 ** 0.5)
                put(a + n + ".bias", 0.05 * torch.randn(512, generator=g, device=self.device))
            norm("encoder.conv_norm_out", 512)
            conv("encoder.conv_out", 32, 512, 3)
            if self._lib.rf_vae_missing_weights(self._h) != 0:
                L.check(-4, "init_synthetic_weights")
        return self

    @torch.no_grad()
    def decode_packed(self, packed_latents: torch.Tensor, height: int, width: int, output: str = "u8"):
        """packed_latents [B, (h/16)(w/16), 64] -> uint8 [B, H, W, 3] (output='u8') or bf16
        [B, 3, H, W] (output='pt')."""
        lat = packed_latents.detach().to(self.device, torch.bfloat16).contiguous()
        B = lat.shape[0]
        u8 = torch.empty((B, height, width, 3), dtype=torch.uint8, device=self.device) if output == "u8" else None
        pt = torch.empty((B, 3, height, width), dtype=torch.bfloat16, device=self.device) if output == "pt" else None
        with torch.cuda.device(self.device):
            for b in range(B):
                L.check(self._lib.rf_vae_decode(
                    self._h, L.ptr(lat[b]), height, width, ctypes.c_float(self.config.scaling_factor),
                    ctypes.c_float(self.config.shift_factor), L.ptr(u8[b]) if u8 is not None else None,
                    L.ptr(pt[b]) if pt is not None else None, L.cur_stream()), "rf_vae_decode")
        return u8 if output == "u8" else pt


    @torch.no_grad()
    def _encode(self, image_u8=None, image_pt=None, eps: Optional[torch.Tensor] = None):
        if image_u8 is not None:
            img = image_u8.detach().to(self.device, torch.uint8).contiguous()
            B, H, W = img.shape[0], img.shape[1], img.shape[2]
        else:
            img = image_pt.detach().to(self.device, torch.bfloat16).contiguous()
            B, H, W = img.shape[0], img.shape[2], img.shape[3]
        out = torch.empty((B, (H // 16) * (W // 16), 64), dtype=torch.bfloat16, device=self.device)
        if eps is not None:
            eps = eps.detach().to(self.device, torch.bfloat16).contiguous()
            if eps.dim() == 3:
                eps = eps[None].expand(B, -1, -1, -1).contiguous()
        with torch.cuda.device(self.device):
            for b in range(B):
                L.check(self._lib.rf_vae_encode(
                    self._h, L.ptr(img[b]) if image_u8 is not None else None,
                    L.ptr(img[b]) if image_u8 is None else None, H, W,
                    L.ptr(eps[b]) if eps is not None else None,
                    ctypes.c_float(self.config.scaling_factor), ctypes.c_float(self.config.shift_factor),
                    L.ptr(out[b]), L.cur_stream()), "rf_vae_encode")
        return out

    def encode_packed(self, image_u8: torch.Tensor, eps: Optional[torch.Tensor] = None):
        """uint8 [B, H, W, 3] -> packed condition tokens [B, (H/16)(W/16), 64] (encode_images of
        train_flux/flux/pipeline_tools.py:7-30).  eps: bf16 [16, H/8, W/8] posterior noise (the
        reference samples it from the global RNG); None = posterior mode."""
        return self._encode(image_u8=image_u8, eps=eps)

    def encode_packed_pt(self, image_pt: torch.Tensor, eps: Optional[torch.Tensor] = None):
        """bf16 [B, 3, H, W] in [-1, 1] (already preprocessed) -> packed tokens."""
        return self._encode(image_pt=image_pt, eps=eps)


def to_pil(u8: torch.Tensor) -> List:
    """uint8 [B, H, W, 3] -> list of PIL images (VaeImageProcessor.numpy_to_pil)."""
    from PIL import Image
    arr = u8.cpu().numpy()
    return [Image.fromarray(a) for a in arr]
