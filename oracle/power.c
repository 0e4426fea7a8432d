/* ORACLE (test infrastructure): SPEC PW, the power inspector.  See power.h. */
#include "power.h"

void sdo_power_init(sdo_power *p, uint64_t M)
{
  p->M = M ? M : 1;
  p->acc = p->c = 0.0;
  p->n = 0;
}

size_t sdo_power_feed(sdo_power *p, const sdo_cpx *x, size_t m, float *mean)
{
  size_t k = 0;
  for (size_t i = 0; i < m; ++i) {
    /* PW.1: Re(x conj(x)) = re re - im (-im): two rounded products and one rounded sum (no contraction) */
    const float pw = x[i].re * x[i].re + x[i].im * x[i].im;
    /* PW.2: Kahan step, RMSInspector.cpp:551-556 */
    const double y = (double) pw - p->c;
    const double t = p->acc + y;
    p->c = (t - p->acc) - y;
    p->acc = t;
    ++p->n;
    /* PW.3: RMSInspector.cpp:329-336 */
    if (p->n >= p->M) {
      mean[k++] = (float) (p->acc / (double) p->n);
      p->acc = p->c = 0.0;
      p->n = 0;
    }
  }
  return k;
}
