// Host build of the loss-option criterion of efficientteacher_b200/csrc/loss_math.h (positive-weight BCE and focal
// loss, value and hand-written derivative) for the CPU unit test.  Test infrastructure only.
#include "../../efficientteacher_b200/csrc/loss_math.h"
extern "C" void hm_det_bce(const float* x, const float* z, int n, float pw, float gamma, float* val, float* grad) {
  for (int i = 0; i < n; ++i) {
    val[i] = etb_det_bce(x[i], z[i], pw, gamma);
    grad[i] = etb_det_bce_grad(x[i], z[i], pw, gamma);
  }
}
