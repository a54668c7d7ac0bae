"""High-precision truth for the binomial tail P[Bin(n, r) >= x] (the p-value of dist and screen).

The tail is summed directly in mpmath at 60 significant digits, for the exact binary value of the double `r`: whichever
tail is smaller is summed term by term with the ratio recurrence, from a first term computed with `loggamma`, and the
upper tail is 1 minus the lower one where that is the smaller.  mpmath's `betainc` is not used: its hypergeometric series
fails to converge around n = 1e4.  Exponents are unbounded, so results far below the double range are exact too."""
import mpmath as mp

DPS = 60


def _pmf(k, r, n):
    """C(n, k) r^k (1-r)^(n-k) for 0 <= k <= n, at the working precision."""
    lg = mp.loggamma(n + 1) - mp.loggamma(k + 1) - mp.loggamma(n - k + 1)
    return mp.exp(lg + k * mp.log(r) + (n - k) * mp.log1p(-r))


def upper_tail(x, r, n):
    """P[Bin(n, r) >= x] as an mpf with DPS significant digits; r is taken as the exact value of the double it is."""
    x, n = int(x), int(n)
    if x <= 0:
        return mp.mpf(1)
    if x > n:
        return mp.mpf(0)
    with mp.workdps(DPS):
        r = mp.mpf(float(r))                     # mpf(float) is exact
        if r <= 0:
            return mp.mpf(0)
        if r >= 1:
            return mp.mpf(1)
        eps = mp.mpf(10) ** (-DPS - 5)
        odds = r / (1 - r)
        if x > n * r:                            # x above the mean: the upper tail, terms fall from x upwards
            t = _pmf(x, r, n)
            s = t
            for k in range(x, n):
                t *= mp.mpf(n - k) / (k + 1) * odds
                s += t
                if t < s * eps:
                    break
            return +s
        t = _pmf(x - 1, r, n)                    # at or below the mean: 1 - P[X <= x-1], terms fall from x-1 downwards
        s = t
        for k in range(x - 1, 0, -1):
            t *= mp.mpf(k) / (n - k + 1) / odds
            s += t
            if t < s * eps:
                break
        return 1 - s


def upper_tail_float(x, r, n):
    return float(upper_tail(x, r, n))


def grid_x(n, r):
    """The x of the large-n grid for P[Bin(n, r) >= x]: 1, 2, n-1, n and the mean plus {-3, -1, 0, 1, 3, 10, 30, 100}
    standard deviations, clipped to [1, n]."""
    mean = n * r
    sd = (n * r * (1 - r)) ** 0.5
    xs = {1, 2, n - 1, n}
    for z in (-3, -1, 0, 1, 3, 10, 30, 100):
        xs.add(min(n, max(1, int(round(mean + z * sd)))))
    return sorted(x for x in xs if 1 <= x <= n)


GRID_N = (4096, 10000, 28151, 28152, 32768, 100000)
GRID_R = (1e-9, 1e-6, 1e-3, 0.01, 0.05, 0.1, 0.25, 1 / 3, 0.5, 0.63, 0.8, 0.9, 0.99, 0.999)
