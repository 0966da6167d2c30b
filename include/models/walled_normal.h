/* walled_normal.h — a standard normal behind a wall, for the sampler's handling of non-finite log densities
 * (evaluate_ℓ, hamiltonian.jl:202-217; logdensity :251-256; leapfrog's @argcheck :276; divergent leaves NUTS.jl:148-159).
 *   q_0 >= a:  l = -1/2 sum q_i^2,  grad = -q                (dhmc_std_*, so family 0 bit for bit)
 *   q_0 <  a:  what a model without a transform returns beyond its support, chosen by `mode`:
 *     0  l = -Inf,  grad = -q          (the ordinary wall: rejected, also by a strict evaluation)
 *     1  l = -Inf,  grad_0 = NaN       (still accepted: l == -Inf wins over the gradient)
 *     2  l = NaN,   grad = -q
 *     3  l = +Inf,  grad = -q
 *     4  l finite (the normal's),  grad_0 = NaN
 *     5  l finite,  grad_0 = +Inf
 *     6  l finite,  grad_0 = -Inf
 * params: [a, mode]. */
#define DHMC_USER_NAME "walled_normal"
#define DHMC_USER_NSUMS 1      /* S[0] = sum q_i^2 */

DHMC_HD void dhmc_user_terms(int i, int D, const double* q, const double* params, double* t) {
  (void)D; (void)params;
  t[0] = dhmc_std_term(q[i]);
}
DHMC_HD double dhmc_user_logdensity(int D, const double* q, const double* S, const double* params) {
  (void)D;
  const double l = dhmc_std_lq(S[0]);
  if (q[0] >= params[0]) return l;
  switch ((int)params[1]) {
    case 0: case 1: return -dm_inf();
    case 2: return dm_nan();
    case 3: return dm_inf();
    default: return l;
  }
}
DHMC_HD double dhmc_user_grad(int i, int D, const double* q, const double* S, const double* params) {
  (void)D; (void)S;
  const double g = dhmc_std_grad(q[i]);
  if (i != 0 || q[0] >= params[0]) return g;
  switch ((int)params[1]) {
    case 1: case 4: return dm_nan();
    case 5: return dm_inf();
    case 6: return -dm_inf();
    default: return g;
  }
}
