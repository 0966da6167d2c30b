/* eight_schools_gq.h — eight_schools.h with generated quantities (include/dhmc_models.h): the quantities the analyst
 * reports, on the scale of the centred model, next to the non-centred coordinates the sampler runs in.
 *   G = J + 1 = D - 1:  tau = exp(q_1),  theta_j = mu + tau eta_j = q_0 + tau q_{j+2}   (j = 1..J)
 * Sampling is that of eight_schools.h, bit for bit. */
#include "eight_schools.h"
#undef DHMC_USER_NAME
#define DHMC_USER_NAME "eight_schools_gq"
#define DHMC_USER_GENERATED 1

DHMC_HD int dhmc_user_ngq(int D) { return D - 1; }
DHMC_HD double dhmc_user_generated(int k, int D, const double* q, const double* params) {
  (void)D; (void)params;
  const double tau = dm_exp(q[1]);
  return k == 0 ? tau : q[0] + tau * q[k + 1];
}
