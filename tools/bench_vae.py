#!/usr/bin/env python
"""VAE decode / encode timing at given image sizes, with seeded inputs.

    python tools/bench_vae.py [--sizes 1024x1024,768x1344] [--encode-sizes 512x512] [--iters 5] [--dump DIR]

Prints one JSON line per size, then a per-kernel profile of the first decode size.  TFLOP/s counts the
convolution and attention MACs of diffusers' AutoencoderKL at that size (vae_flops).  --dump DIR writes the
uint8 / bf16 decode outputs and the packed encode output of every size as .npy (bf16 as its uint16 bits), so two
builds can be compared byte for byte; it only uses B200AutoencoderKL, so it runs against older builds too."""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from reflectionflow_b200 import _lib as L  # noqa: E402
from reflectionflow_b200.vae import B200AutoencoderKL  # noqa: E402


def vae_flops(height: int, width: int, decode: bool = True) -> float:
    """2 x MACs of the AutoencoderKL decoder (packed latents -> image) or encoder (image -> moments)"""
    macs = 0.0

    def conv(h, w, cin, cout, taps=9):
        nonlocal macs
        macs += float(h) * w * cin * cout * taps

    def resnet(h, w, cin, cout):
        conv(h, w, cin, cout)
        conv(h, w, cout, cout)
        if cin != cout:
            conv(h, w, cin, cout, 1)

    def mid(h, w):
        nonlocal macs
        n = h * w
        resnet(h, w, 512, 512)
        macs += float(n) * 512 * 512 * 4 + 2.0 * n * n * 512  # q, k, v, out projections; QK^T and PV
        resnet(h, w, 512, 512)

    h, w = height // 8, width // 8
    if decode:
        conv(h, w, 16, 512)
        mid(h, w)
        prev = 512
        for i, c in enumerate((512, 512, 256, 128)):
            for j in range(3):
                resnet(h, w, prev if j == 0 else c, c)
            prev = c
            if i < 3:
                h, w = 2 * h, 2 * w
                conv(h, w, c, c)
        conv(h, w, 128, 3)
    else:
        h, w = height, width
        conv(h, w, 3, 128)
        prev = 128
        for i, c in enumerate((128, 256, 512, 512)):
            for j in range(2):
                resnet(h, w, prev if j == 0 else c, c)
            prev = c
            if i < 3:
                h, w = h // 2, w // 2
                conv(h, w, c, c)
        mid(h, w)
        conv(h, w, 512, 32)
    return 2.0 * macs


def _sizes(s):
    return [tuple(int(v) for v in hw.split("x")) for hw in s.split(",") if hw]


def _time(fn, iters):
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        out = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters, out


def _save(d, name, t):
    import numpy as np
    t = t.cpu()
    if t.dtype == torch.bfloat16:
        t = t.view(torch.int16)
    np.save(os.path.join(d, name + ".npy"), t.numpy())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1024x1024", help="decode sizes HxW, comma separated")
    ap.add_argument("--encode-sizes", default="512x512", help="encode sizes HxW, comma separated")
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--dump", default=None, help="directory for the outputs as .npy")
    ap.add_argument("--no-profile", action="store_true")
    args = ap.parse_args()
    if args.dump:
        os.makedirs(args.dump, exist_ok=True)
    vae = B200AutoencoderKL().init_synthetic_weights(0)
    dev = torch.cuda.get_device_name(0)
    results = []
    for (H, W) in _sizes(args.sizes):
        g = torch.Generator().manual_seed(H * 100003 + W)
        lat = torch.randn(1, (H // 16) * (W // 16), 64, generator=g).to(torch.bfloat16).cuda()
        ms, u8 = _time(lambda: vae.decode_packed(lat, H, W, "u8"), args.iters)
        fl = vae_flops(H, W, True)
        r = {"op": "decode", "height": H, "width": W, "ms": round(ms, 3), "tflops": round(fl / ms / 1e9, 1),
             "ns_per_pixel": round(ms * 1e6 / (H * W), 3), "mean_u8": float(u8.float().mean()), "device": dev}
        if args.dump:
            _save(args.dump, f"decode_u8_{H}x{W}", u8)
            _save(args.dump, f"decode_bf16_{H}x{W}", vae.decode_packed(lat, H, W, "pt"))
        print(json.dumps(r), flush=True)
        results.append(r)
    for (H, W) in _sizes(args.encode_sizes):
        g = torch.Generator().manual_seed(H * 100019 + W)
        img = torch.randint(0, 256, (1, H, W, 3), generator=g, dtype=torch.uint8).cuda()
        eps = torch.randn(16, H // 8, W // 8, generator=g).to(torch.bfloat16)
        ms, packed = _time(lambda: vae.encode_packed(img, eps), args.iters)
        fl = vae_flops(H, W, False)
        r = {"op": "encode", "height": H, "width": W, "ms": round(ms, 3), "tflops": round(fl / ms / 1e9, 1),
             "ns_per_pixel": round(ms * 1e6 / (H * W), 3), "device": dev}
        if args.dump:
            _save(args.dump, f"encode_packed_{H}x{W}", packed)
        print(json.dumps(r), flush=True)
        results.append(r)
    if args.no_profile or not results or results[0]["op"] != "decode":
        return
    H, W = results[0]["height"], results[0]["width"]
    lat = torch.randn(1, (H // 16) * (W // 16), 64, generator=torch.Generator().manual_seed(1)).to(
        torch.bfloat16).cuda()
    L.profile_start()
    vae.decode_packed(lat, H, W, "u8")
    prof = L.profile_stop()
    tot = sum(v["ms"] for v in prof.values())
    for k, v in sorted(prof.items(), key=lambda kv: -kv[1]["ms"]):
        tf = v["flops"] / v["ms"] / 1e9 if v["flops"] else 0
        gb = v["bytes"] / v["ms"] / 1e6
        print(f"  {k:16s} launches {v['launches']:3d}  ms {v['ms']:7.3f}  share {v['ms']/tot:.3f}  {tf:7.1f} TF/s  "
              f"{gb:7.1f} GB/s")


if __name__ == "__main__":
    main()
