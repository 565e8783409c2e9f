"""Host emulation of sample_noise_kernel (TEST INFRASTRUCTURE; tests/emu_core.py): the kernel's text (csrc/reduce.cu,
``[emu:... noise]``) and the xoroshiro128+ step (csrc/common.cuh) compiled with g++.  logf / cosf are libm's (the GPU
uses libdevice's, both within an ulp or two), sqrt.approx becomes sqrtf.  The kernel has no barriers: its threads run
one after the other."""
from tests.emu_core import build as _build
from tests.emu_core import region

HARNESS = r'''
extern "C" void emu_sample_noise(uint64_t* states, float* noise, long long count, float std_v, float std_w, float* reach) {
  emu::launch_serial({(unsigned)((count + 255) / 256), 1, 1}, 256, [&] {
    b200::sample_noise_kernel(states, reinterpret_cast<float2*>(noise), count, std_v, std_w, reach);
  });
}
'''


def build(out_dir, extra=""):
    parts = [region("common.cuh", "xoro"), region("common.cuh", "normal"), region("reduce.cu", "noise")]
    return _build(out_dir, "noise_emu", parts, HARNESS + extra)
