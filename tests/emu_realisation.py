"""Host emulation of the ground-truth realisation conversion (TEST INFRASTRUCTURE; tests/emu_core.py):
realisation_convert_kernel, text lifted from csrc/sample.cu, with its argument struct from kernels.h.  No barriers:
threads run one after the other, and the float32 operations are the host's IEEE ones (no flush to zero)."""
from tests.emu_core import build as _build
from tests.emu_core import region

HARNESS = r'''
using namespace b200;
// planes 1 or 2: plane p converts grid[p] (rows of pitch[p] bytes, bounds lo[p], hi[p]) into out[p] (rows, cols)
extern "C" void emu_realisation_convert(const int8_t** grid, const int* pitch, const float* lo, const float* hi,
                                        double** out, int planes, int rows, int cols) {
  RealisationPlane p[2];
  for (int i = 0; i < 2; ++i) {
    const int j = i < planes ? i : 0;
    p[i] = RealisationPlane{grid[j], pitch[j], lo[j], hi[j], out[j]};
  }
  const long long cells = (long long)rows * cols;
  emu::launch_serial({(unsigned)((cells + 255) / 256), (unsigned)planes, 1}, 256,
                     [&] { realisation_convert_kernel(p[0], p[1], rows, cols); });
}
'''


def build(out_dir):
    return _build(out_dir, "realisation_emu", [region("kernels.h", "realisation_args"), region("sample.cu", "realisation")],
                  HARNESS)
