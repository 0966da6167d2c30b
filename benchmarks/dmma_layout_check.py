"""Round-2 preparation for the FP64-MMA version of the cooperative logistic likelihood
(DESIGN.md §7 (i)): checks, on the CPU, the two things that are easy to get wrong when writing
the kernel — the m8n8k4 fragment index formulas for both phases, and that the planned
shared-memory strides make every fragment load bank-conflict free.

The MMA itself is emulated with the accumulation order that benchmarks/dmma_order_probe.cu checks on
the device: d = fma(a3,b3, fma(a2,b2, fma(a1,b1, fma(a0,b0, c)))).
Run: python benchmarks/dmma_layout_check.py"""
from fractions import Fraction

import numpy as np


def fma(a, b, c):
    """Correctly rounded a·b + c (Fraction arithmetic is exact, float() rounds to nearest even)."""
    return float(Fraction(float(a)) * Fraction(float(b)) + Fraction(float(c)))

G = 8                      # chains per CTA = the n-dimension of the MMA


def mma_m8n8k4(a_frag, b_frag, c_frag):
    """One warp-wide mma.sync.m8n8k4.f64.  a_frag[lane] = A[lane>>2][lane&3], b_frag[lane] =
    B[lane&3][lane>>2], c_frag[lane] = (C[lane>>2][2(lane&3)], C[lane>>2][2(lane&3)+1])."""
    A = np.empty((8, 4)); B = np.empty((4, 8)); C = np.empty((8, 8))
    for lane in range(32):
        A[lane >> 2, lane & 3] = a_frag[lane]
        B[lane & 3, lane >> 2] = b_frag[lane]
        C[lane >> 2, 2 * (lane & 3)], C[lane >> 2, 2 * (lane & 3) + 1] = c_frag[lane]
    D = C.copy()
    for i in range(8):
        for j in range(8):
            acc = C[i, j]
            for k in range(4):
                acc = fma(A[i, k], B[k, j], acc)
            D[i, j] = acc
    return [(D[lane >> 2, 2 * (lane & 3)], D[lane >> 2, 2 * (lane & 3) + 1]) for lane in range(32)]


def conflict_free_64(addresses):
    """LDS.64 of a warp = two half-warp wavefronts; a wavefront is conflict free if its 16
    addresses (in doubles) fall into 16 different 8-byte bank pairs."""
    a = np.asarray(addresses)
    return all(len({int(x) % 16 for x in a[h * 16:(h + 1) * 16]}) == 16 for h in range(2))


def phase1(N, p, seed=0):
    """η[n][g] = Σ_j X[n][j] β[g][j]: A = 8 observations × 4 coefficients from the Xᵀ ring tile
    (row stride RS ≡ 4 mod 16), B = β stored [chain][p + pad] with the same stride rule."""
    rng = np.random.default_rng(seed)
    X, beta = rng.normal(size=(N, p)), rng.normal(size=(G, p))
    ref = np.empty((N, G))
    for n in range(N):
        for g in range(G):
            acc = 0.0
            for j in range(p):
                acc = fma(X[n, j], beta[g, j], acc)
            ref[n, g] = acc
    pk = (p + 3) // 4 * 4
    RB = 32                                   # observations of this toy tile
    RS = RB + 4                               # ≡ 4 mod 16 for RB ≡ 0 mod 16
    BS = pk                                   # row stride of β, padded up to ≡ 4 mod 16
    while BS % 16 != 4:
        BS += 1
    bsm = np.zeros(G * BS)
    for g in range(G):
        bsm[g * BS:g * BS + p] = beta[g]      # k-padding of β is zero
    eta = np.zeros((N, G))
    ok = True
    for n0 in range(0, N, RB):
        for rt in range(RB // 8):             # one 8-row tile = one MMA per k-step
            c = [(0.0, 0.0)] * 32
            for j0 in range(0, pk, 4):
                tile = np.zeros(4 * RS)       # ring tile: rows j0..j0+3 of Xᵀ, zero beyond p / N
                for jj in range(4):
                    for r in range(RB):
                        if j0 + jj < p and n0 + r < N:
                            tile[jj * RS + r] = X[n0 + r, j0 + jj]
                a_addr = [(lane & 3) * RS + rt * 8 + (lane >> 2) for lane in range(32)]
                b_addr = [(lane >> 2) * BS + j0 + (lane & 3) for lane in range(32)]
                ok &= conflict_free_64(a_addr) and conflict_free_64(b_addr)
                c = mma_m8n8k4([tile[x] for x in a_addr], [bsm[x] for x in b_addr], c)
            for lane in range(32):
                n = n0 + rt * 8 + (lane >> 2)
                if n < N:
                    eta[n, 2 * (lane & 3)], eta[n, 2 * (lane & 3) + 1] = c[lane]
    return np.array_equal(eta, ref), ok


def phase2(N, p, seed=1):
    """(Xᵀr)[j][g] = Σ_n X[n][j] r[n][g]: A = 8 coefficients × 4 observations from the X ring tile
    (row stride p + pad ≡ 4 mod 16), B = residuals stored [n][G + 4]."""
    rng = np.random.default_rng(seed)
    X, r = rng.normal(size=(N, p)), rng.normal(size=(N, G))
    ref = np.empty((p, G))
    for j in range(p):
        for g in range(G):
            acc = 0.0
            for n in range(N):
                acc = fma(X[n, j], r[n, g], acc)
            ref[j, g] = acc
    XS = p
    while XS % 16 != 4:
        XS += 1
    RSr = G + 4                                # 12: k·12 + g distinct mod 16 for k, g < 4
    Nk = (N + 3) // 4 * 4
    xs = np.zeros(Nk * XS); rs = np.zeros(Nk * RSr)   # zero-filled k-padding (n >= N)
    for n in range(N):
        xs[n * XS:n * XS + p] = X[n]
        rs[n * RSr:n * RSr + G] = r[n]
    out = np.zeros((p, G))
    ok = True
    for jt in range((p + 7) // 8):
        c = [(0.0, 0.0)] * 32
        for n0 in range(0, Nk, 4):
            a_addr = [(n0 + (lane & 3)) * XS + jt * 8 + (lane >> 2) for lane in range(32)]
            b_addr = [(n0 + (lane & 3)) * RSr + (lane >> 2) for lane in range(32)]
            ok &= conflict_free_64(a_addr) and conflict_free_64(b_addr)
            a = [xs[x] if jt * 8 + (lane >> 2) < p else 0.0 for lane, x in enumerate(a_addr)]
            c = mma_m8n8k4(a, [rs[x] for x in b_addr], c)
        for lane in range(32):
            j = jt * 8 + (lane >> 2)
            if j < p:
                out[j, 2 * (lane & 3)], out[j, 2 * (lane & 3) + 1] = c[lane]
    return np.array_equal(out, ref), ok


if __name__ == "__main__":
    for N, p in ((64, 16), (50, 13), (96, 40)):
        e1, b1 = phase1(N, p)
        e2, b2 = phase2(N, p)
        print(f"N={N} p={p}: phase 1 bit-exact={e1} conflict-free={b1}; phase 2 bit-exact={e2} conflict-free={b2}")
        assert e1 and b1 and e2 and b2
    print("fragment formulas and shared-memory strides check out")
