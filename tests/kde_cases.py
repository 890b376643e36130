"""Restatement of est_kernel_density's arithmetic (scipy.stats.gaussian_kde with
bw_method = bw / std(ddof=1), evaluated on a grid) and the bounds the device is held to
(DESIGN.md §2 "Kernel densities").  No GPU and no reference tree needed."""
import math

import numpy as np
from scipy import stats

U = 2.0 ** -53
TINY = 2.0 ** -1074


def gamma(n):
    return n * U / (1 - n * U)


def factor_of(x, bw):
    """bw / x.std(ddof=1): numpy's pairwise sums"""
    return bw / np.asarray(x, dtype=np.float64).std(ddof=1)


def cho_cov_pairwise(x, factor):
    """sqrt(np.cov(x, aweights=ones(n)/n)) * factor with np.cov's BLAS dot replaced by a
    numpy pairwise sum (the device's c, bit for bit)"""
    x = np.asarray(x, dtype=np.float64)
    w = np.ones(x.shape[0]) / x.shape[0]
    w_sum = np.sum(w)
    avg = np.sum(x * w) / w_sum
    fact = w_sum - 1 * np.sum(w * w) / w_sum
    d = x - avg
    return math.sqrt(np.sum(d * (d * w)) * (1.0 / fact)) * factor


def c_bound(n):
    """relative bound |c_device - c_scipy| / c_scipy: both dots of non-negative terms within
    gamma_n of the exact one (the square root halves that), then 1/fact, sqrt and * factor
    round on each side"""
    return gamma(n) + 6 * U


def restate_kde(x, grid, c):
    """gaussian_kernel_estimate at kernel width c, term by term with libm exp (math.exp),
    summed sequentially in data order -- bit-identical to gaussian_kde.evaluate"""
    x, grid = np.asarray(x, dtype=np.float64), np.asarray(grid, dtype=np.float64)
    w = np.ones(x.shape[0]) / x.shape[0]
    inv = 1 / c
    p, q = x * inv, grid * inv
    norm = math.pow(2 * math.pi, -0.5) / c
    exp = np.frompyfunc(math.exp, 1, 1)
    d = np.zeros(grid.shape[0])
    with np.errstate(under='ignore'):
        for i in range(x.shape[0]):
            a = (p[i] - q) * (p[i] - q)
            d += w[i] * (exp(-a / 2.).astype(np.float64) * norm)
    return d


def scipy_kde(x, grid, bw):
    """(densities, cho_cov) of the reference's call"""
    x = np.asarray(x, dtype=np.float64)
    kde = stats.gaussian_kde(x, bw_method=bw / x.std(ddof=1))
    with np.errstate(under='ignore'):
        return kde.evaluate(grid), float(kde.cho_cov[0, 0])


def scipy_kde_at(x, grid, c):
    """scipy's own evaluation with the kernel width set to c (the restatement at c, fast)"""
    x = np.asarray(x, dtype=np.float64)
    kde = stats.gaussian_kde(x)
    kde.cho_cov = np.array([[c]])
    with np.errstate(under='ignore'):
        return kde.evaluate(grid)


def density_bound(x, grid, c, ref):
    """|D_j - R_j| for the device's D and the restatement R at the same c:
    (9 u + gamma_{n-1} + gamma_{ceil(n/8)+3}) sum_i t_ij + (n + norm) 2^-1072.
    9 u: each term's exp is within 1 ulp (2 u relative) in either library, and its two
    products round on each side; the sums: sequential on the host, 8 sequential stripes and a
    3-level tree on the device.  sum_i t_ij <= R_j (1 + gamma_{n-1}) since every t >= 0."""
    n = np.asarray(x).shape[0]
    norm = math.pow(2 * math.pi, -0.5) / c
    g = gamma(n - 1)
    return ((9 * U + g + gamma(-(-n // 8) + 3)) * ref * (1 + g) + (n + norm) * TINY * 4)


def c_widening(x, grid, c, c_ref):
    """|R_j(c) - R_j(c_ref)|, the restatement at two kernel widths.  Two parts per term:
    - the exact change: dt/dc = t (a - 1) / c with a = (x - g)^2 / c^2, at most
      2 rho |a - 1| t for rho = |c - c_ref| / c_ref << 1 / max a;
    - the whitening: p = x * (1 / c) and q = g * (1 / c) round differently at the two
      widths, each within 2 u of x / c and g / c, so d = p - q moves by at most
      2 u (|p| + |q|) on each side, and t (proportional to exp(-d^2 / 2)) by |d| times that."""
    x, grid = np.asarray(x, dtype=np.float64), np.asarray(grid, dtype=np.float64)
    rho = abs(c - c_ref) / c_ref
    out = np.zeros(grid.shape[0])
    norm = math.pow(2 * math.pi, -0.5) / c_ref
    with np.errstate(under='ignore'):
        for lo in range(0, x.shape[0], 256):
            xs = x[lo:lo + 256, None]
            d = (xs - grid[None, :]) / c_ref
            a = d * d
            t = np.exp(-a / 2) * norm / x.shape[0]
            whiten = 4 * U * (np.abs(xs) + np.abs(grid[None, :])) / c_ref * np.abs(d)
            out += ((2 * rho * np.abs(a - 1) + whiten) * t).sum(axis=0)
    return out * 1.01


def seeded_sets():
    """(levels, grid, bw) cases: n = 2 .. 4000, bw 0.01 .. 0.5, and data at the grid's edge
    so the far tail underflows"""
    rs = np.random.RandomState(1914)
    grid = np.linspace(-5, 5, 200)
    cases = []
    for n, bw, loc, sd in ((2, 0.05, 0.0, 1.0), (3, 0.5, 1.0, 0.3), (7, 0.01, -2.0, 0.5),
                           (129, 0.2, 0.0, 1.0), (1000, 0.05, 4.9, 0.05),
                           (4000, 0.3, -1.0, 0.8), (500, 0.01, -4.95, 0.02), (64, 0.1, 0.0, 2.0)):
        cases.append((rs.normal(loc, sd, n), grid, bw))
    return cases
