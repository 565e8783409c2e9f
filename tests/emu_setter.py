"""Host emulation of the setter kernels (TEST INFRASTRUCTURE; tests/emu_core.py): build_cum_kernel (the cumulative
table the sampler reads) and collapse_pad_kernel (CVaR / mean collapse + crop + padding of the one-map modes), text
lifted from csrc/sample.cu.  No barriers in these kernels: threads run one after the other."""
from tests.emu_core import build as _build
from tests.emu_core import region

HARNESS = r'''
static EmuDim3 blocks_for(long long threads_total) { return {(unsigned)((threads_total + 255) / 256), 1, 1}; }
extern "C" void emu_build_cum(const int8_t* pmf, int8_t* cum, int B, int bpad, int rows, int cols) {
  emu::launch_serial(blocks_for((long long)rows * cols), 256, [&] { b200::build_cum_kernel(pmf, cum, B, bpad, rows, cols); });
}
extern "C" void emu_collapse_pad(const int8_t* raw, int8_t* out, int8_t* risk, int* bad, const float* bin_values, int B,
                                 int H, int W, int keep_r, int keep_c, int pad, int risk_pitch, double alpha, float lo,
                                 float range, int mode) {
  emu::launch_serial(blocks_for((long long)(keep_r + 2 * pad) * (keep_c + 2 * pad)), 256, [&] {
    b200::collapse_pad_kernel(raw, out, risk, bad, bin_values, B, H, W, keep_r, keep_c, pad, risk_pitch, alpha, lo, range,
                              mode);
  });
}
'''


def build(out_dir, extra=""):
    return _build(out_dir, "setter_emu", [region("sample.cu", "build_cum"), region("sample.cu", "collapse_pad")],
                  HARNESS + extra)
