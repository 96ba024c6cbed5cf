"""not-gpu: the C-ABI shared library loads and exports every symbol include/rf_b200.h declares;
without a GPU the compute entry points fail loudly (no CPU fallback)."""
import ctypes
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    src = open(os.path.join(ROOT, "include", "rf_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(rf_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    from reflectionflow_b200 import _lib
    lib = _lib.load()
    names = _declared()
    assert "rf_dit_forward" in names and "rf_op_linear" in names and len(names) >= 18
    for n in names:
        assert hasattr(lib, n), f"{n} declared in include/rf_b200.h but not exported"
    assert lib.rf_abi_version() == 2


def test_sass_is_hopper_native():
    """the shipped binary is sm_90a code whose tensor-core work is wgmma (HGMMA) fed by TMA (UTMALDG)."""
    import shutil
    import subprocess
    if not shutil.which("cuobjdump"):
        pytest.skip("cuobjdump not on PATH")
    so = os.path.join(ROOT, "reflectionflow_b200", "librf_b200.so")
    sass = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True).stdout
    archs = set(re.findall(r"arch = (sm_\w+)", sass))
    assert archs == {"sm_90a"}, archs
    for mnem in ("HGMMA.", "UTMALDG", "SYNCS."):
        assert mnem in sass, mnem
    assert "HMMA." not in sass.replace("HGMMA.", ""), "legacy mma.sync path must not be present"


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU failure mode")
def test_no_gpu_fails_loudly():
    from reflectionflow_b200 import _lib
    from reflectionflow_b200.transformer import B200FluxTransformer2DModel
    with pytest.raises(_lib.RFError):
        B200FluxTransformer2DModel()
    lib = _lib.load()

    class Cfg(ctypes.Structure):
        _fields_ = [(n, ctypes.c_int) for n in ("a", "b", "c", "d", "e", "f", "g", "h")]
    cfg = Cfg(1, 1, 2, 64, 128, 64, 1, 0)
    h = ctypes.c_void_p()
    rc = lib.rf_dit_create(ctypes.byref(cfg), ctypes.byref(h))
    assert rc != 0 and b"no CUDA device" in lib.rf_last_error()


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU failure mode")
def test_no_gpu_fails_loudly_vae_and_text():
    from reflectionflow_b200 import _lib
    from reflectionflow_b200.text import B200TextEncoders
    from reflectionflow_b200.vae import B200AutoencoderKL
    with pytest.raises(_lib.RFError):
        B200TextEncoders()
    with pytest.raises(_lib.RFError):
        B200AutoencoderKL()
    lib = _lib.load()
    from reflectionflow_b200.text import _TextCfg, T5_XXL, CLIP_L
    cfg = _TextCfg(**dict(T5_XXL, **CLIP_L))
    h = ctypes.c_void_p()
    assert lib.rf_text_create(ctypes.byref(cfg), ctypes.byref(h)) != 0
    assert b"no CUDA device" in lib.rf_last_error()


def _build_c_example(tmp_path):
    import shutil
    import subprocess
    if not shutil.which("gcc"):
        pytest.skip("gcc not on PATH")
    cuda = os.environ.get("CUDA_HOME", "/usr/local/cuda")
    exe = str(tmp_path / "c_abi_linear")
    libdir = os.path.join(ROOT, "reflectionflow_b200")
    cmd = ["gcc", "-std=c11", "-O2", "-Wall", "-Werror", "-I" + os.path.join(ROOT, "include"),
           "-I" + os.path.join(cuda, "include"), os.path.join(ROOT, "examples", "c_abi_linear.c"),
           "-L" + libdir, "-lrf_b200", "-L" + os.path.join(cuda, "lib64"), "-lcudart", "-lm",
           "-Wl,-rpath," + libdir, "-o", exe]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return exe


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU failure mode")
def test_c_example_builds_against_the_header_and_fails_loudly_without_gpu(tmp_path):
    """include/rf_b200.h is plain C11 and the library links from C (no Python, no torch)."""
    import subprocess
    exe = _build_c_example(tmp_path)
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 2 and "no CUDA device" in r.stderr


@pytest.mark.gpu
def test_c_example_linear_matches_scalar_host_loop(tmp_path):
    """rf_op_linear driven from plain C agrees with a scalar host loop (<= 1 bf16 ulp on < 2 % of outputs)."""
    import subprocess
    exe = _build_c_example(tmp_path)
    r = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    print(r.stdout)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "c_abi_linear: OK" in r.stdout
