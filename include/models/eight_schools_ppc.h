/* eight_schools_ppc.h — eight_schools.h with random generated quantities (include/dhmc_models.h): a posterior predictive
 * check.  Rows (J = D - 2, G = 2J + 4 = 2D):
 *   k = 0              tau = exp(q_1)
 *   k = 1 .. J         theta_j = mu + tau eta_j = q_0 + tau q_{j+1}                 (as eight_schools_gq.h)
 *   k = J+1 .. 2J      y_rep_j = theta_j + sigma_j normal(j - 1)                      (j = k - J)
 *   k = 2J+1           1{max_j y_rep_j >= max_j y_j}
 *   k = 2J+2           1{min_j y_rep_j <= min_j y_j}
 *   k = 2J+3           1{chi2(y_rep, theta) >= chi2(y, theta)},  chi2(x, theta) = sum_j ((x_j - theta_j)/sigma_j)^2
 * The three indicators re-derive y_rep through the same indices, so the summary mean of each is a posterior predictive
 * p-value.  Sampling is that of eight_schools.h, bit for bit. */
#include "eight_schools.h"
#undef DHMC_USER_NAME
#define DHMC_USER_NAME "eight_schools_ppc"
#define DHMC_USER_GENERATED 1
#define DHMC_USER_GENERATED_RNG 1

DHMC_HD int dhmc_user_ngq(int D) { return 2 * D; }
DHMC_HD double dhmc_user_generated(int k, int D, const double* q, const double* params, const dhmc_gq_rng* rng) {
  const int J = D - 2;
  const double* y = params;
  const double* sigma = params + J;
  const double tau = dm_exp(q[1]);
  if (k == 0) return tau;
  if (k <= J) return q[0] + tau * q[k + 1];
  if (k <= 2 * J) {
    const int j = k - J - 1;
    return (q[0] + tau * q[j + 2]) + sigma[j] * dhmc_gq_normal(rng, (uint32_t)j);
  }
  double rep_max = -dm_inf(), rep_min = dm_inf(), y_max = -dm_inf(), y_min = dm_inf(), chi_rep = 0.0, chi_y = 0.0;
  for (int j = 0; j < J; ++j) {
    const double theta = q[0] + tau * q[j + 2];
    const double rep = theta + sigma[j] * dhmc_gq_normal(rng, (uint32_t)j);
    const double zr = (rep - theta) / sigma[j], zy = (y[j] - theta) / sigma[j];
    rep_max = rep > rep_max ? rep : rep_max;
    rep_min = rep < rep_min ? rep : rep_min;
    y_max = y[j] > y_max ? y[j] : y_max;
    y_min = y[j] < y_min ? y[j] : y_min;
    chi_rep = chi_rep + zr * zr;
    chi_y = chi_y + zy * zy;
  }
  if (k == 2 * J + 1) return rep_max >= y_max ? 1.0 : 0.0;
  if (k == 2 * J + 2) return rep_min <= y_min ? 1.0 : 0.0;
  return chi_rep >= chi_y ? 1.0 : 0.0;
}
