import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_host_fft_r32_emulation():
    """The 32 x 32 x 16 plan of the 16384-point Float32 overlap-save kernels (fft_r32 in fft_core.cuh) compiled for the
    host and run pass by pass: forward transform and overlap-save pipeline vs a double FFT, bank audit of every pass."""
    exe = os.path.join(ROOT, "build", "fft_r32_host_check")
    os.makedirs(os.path.dirname(exe), exist_ok=True)
    src = os.path.join(ROOT, "tests", "host", "fft_r32_host_check.cu")
    if not os.path.exists(exe) or os.path.getmtime(exe) < max(os.path.getmtime(src), os.path.getmtime(
            os.path.join(ROOT, "dsp.jl_b200", "csrc", "fft_core.cuh"))):
        subprocess.run(["g++", "-std=c++17", "-O2", "-x", "c++", "-w", "-I/usr/local/cuda/include", "-o", exe, src], check=True)
    out = subprocess.run([exe], capture_output=True, text=True)
    assert out.returncode == 0 and "ALL OK" in out.stdout, out.stdout
