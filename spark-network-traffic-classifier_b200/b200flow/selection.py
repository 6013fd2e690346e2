"""Univariate feature selection on the device (DESIGN.md §5i): the chi-square, ANOVA and F-value tests and the variance of
each feature, from csrc/selection.cu's distinct-value, contingency and centred-moment kernels and the grouped-sum kernel,
summed in the chunk order of dist.Shards; the statistics, p-values and selection rules on the host from totals that are the
same bits on every rank.

Spark [recalled; Spark 3.1 `ml/stat/ChiSquareTest.scala`, `mllib/stat/test/ChiSqTest.scala`, `ml/stat/ANOVATest.scala`,
`ml/stat/FValueTest.scala`, `ml/feature/Selector.scala`, `ml/feature/UnivariateFeatureSelector.scala`,
`ml/feature/ChiSqSelector.scala`, `ml/feature/VarianceThresholdSelector.scala`]:

    ChiSquareTest: per feature j the contingency table of its distinct values (Scala ==, so -0.0 and +0.0 are one value)
    against the distinct label values; more than 10000 distinct values in a feature (or the label) raises (maxCategories).
    e = rowSum colSum / n, statistic = sum (o - e)^2 / e, dof = (values - 1)(labels - 1), pValue = 1.0 - ChiSq(dof).cdf(stat);
    dof == 0 gives statistic 0.0 and pValue 1.0.
    ANOVATest (continuous feature, categorical label, k classes): F = (SSB / (k - 1)) / (SSW / (n - k)),
    pValue = 1.0 - F(k - 1, n - k).cdf(F), degreesOfFreedom = n - 1.
    FValueTest (continuous feature and label): F = r^2 / (1 - r^2) (n - 2), r Pearson's r, dof = n - 2,
    pValue = 1.0 - F(1, n - 2).cdf(F).
    Selection (numTopFeatures, percentile, fpr, fdr, fwe): sort by p-value ascending, ties by feature index, NaN last
    (java.lang.Double.compare); numTopFeatures keeps k, percentile keeps (D percentile).toInt; fpr keeps p < fpr; fwe keeps
    p < fwe / D; fdr (Benjamini-Hochberg) keeps the first i + 1 of the sorted list, i the largest index with
    p_(i) <= fdr (i + 1) / D.  A NaN never passes a threshold.  selectedFeatures ascending.
    VarianceThresholdSelector keeps the features whose unbiased variance is > varianceThreshold.

Order of the arithmetic (what makes the result the same bits for any world size):
    the contingency counts are int64 sums; the class sums and counts come from b200flow_group_sums, the centred sums from
    b200flow_group_centered_moments with the class means (or the grand means) as centres, both chained in chunk order.  On
    the host: chi-square sums its (o - e)^2 / e terms sequentially in (value, label) order from +0.0, e = (rowSum colSum) / n;
    ANOVA's mean_g = sum_g / n_g, grand = (sum over g in order of sum_g) / n, SSW = sum over g in order of the centred sums,
    SSB = sum over g in order of n_g (mean_g - grand)^2; F-value's r = Sxy / (sqrt(Sxx) sqrt(Syy)).

Deviations: the centred sums are two-pass, not Spark's raw sum of squares (the same in exact arithmetic; a column near 1e9
keeps its variance); the p-values come from this module's incomplete gamma and beta, not commons-math's; non-finite features
or labels raise ValueError; D <= 256; at most 256 distinct labels for chi-square and ANOVA (Spark allows 10000); a
contingency table set of at most 2^26 cells; ANOVA needs k >= 2 and n > k, F-value n > 2.
"""
import math

import numpy as np
import torch

from . import _lib
from . import dist as bdist
from ._lib import call, ptr

MAX_D = 256
MAX_LABELS = 256
MAX_CATEGORIES = 10000
MAX_CELLS = 1 << 26
TABLE_SLOTS = 1 << 15
# device memory for one batch of chunks' partial rows (at G = 256 classes and D = 256 a partial row is 512 KiB)
PARTIALS_BUDGET = 64 << 20


class TooManyValuesError(ValueError):
    """more than MAX_CATEGORIES distinct values in one column (Spark raises a SparkException)."""


# ----------------------------------------------------------------------------------- special functions
_EPS = 1e-16
_TINY = 1e-300
_MAX_ITER = 10000000
_HALF_LN_2PI = 0.5 * math.log(2.0 * math.pi)
_LN_1E250 = 250.0 * math.log(10.0)


def _stirlerr(z):
    """ln Gamma(z) - ((z - 1/2) ln z - z + ln sqrt(2 pi)), z > 0."""
    if z < 10.0:
        return math.lgamma(z) - (z - 0.5) * math.log(z) + z - _HALF_LN_2PI
    r = 1.0 / z
    r2 = r * r
    return r * (1.0 / 12 - r2 * (1.0 / 360 - r2 * (1.0 / 1260 - r2 * (1.0 / 1680 - r2 * (1.0 / 1188)))))


def _log1pmx(t, q):
    """t - ln(1 + t), t >= -1, q = 1 + t computed separately: a series near 0, where ln(1 + t) would cancel."""
    if abs(t) >= 0.25:
        return t - math.log(q) if q > 0.0 else math.inf
    term, s, k = -t, 0.0, 1
    while True:
        k += 1
        term = -term * t
        d = term / k
        s += d
        if abs(d) <= _EPS * 1e-2 * abs(s):
            return s


def _log_gamma_prefix(a, x):
    """ln(x^a e^-x / Gamma(a)) = -a log1pmx((x - a) / a) + ln sqrt(a / 2 pi) - stirlerr(a): no large terms cancel."""
    return -a * _log1pmx((x - a) / a, x / a) + 0.5 * math.log(a) - _HALF_LN_2PI - _stirlerr(a)


def _log_beta_prefix(x, y, a, b):
    """ln(x^a y^b / B(a, b)), y = 1 - x given separately: -a log1pmx(u) - b log1pmx(v) + ln sqrt(a b / (2 pi (a + b)))
    + stirlerr(a + b) - stirlerr(a) - stirlerr(b), 1 + u = x (a + b) / a, 1 + v = y (a + b) / b.  a u + b v = 0, so u and v
    are both taken from the smaller of x and y: with b ~ 1e6 the other one's rounding alone would move the result by 1e-10."""
    if x <= y:
        qu = x * ((a + b) / a)
        u = (x * (a + b) - a) / a
        v = -(a * u) / b
        qv = 1.0 + v
    else:
        qv = y * ((a + b) / b)
        v = (y * (a + b) - b) / b
        u = -(b * v) / a
        qu = 1.0 + u
    return (-a * _log1pmx(u, qu) - b * _log1pmx(v, qv) + 0.5 * math.log(a * b / (a + b)) - _HALF_LN_2PI
            + _stirlerr(a + b) - _stirlerr(a) - _stirlerr(b))


def gamma_p(a, x):
    """regularised lower incomplete gamma P(a, x): the series below a + 1, else 1 - Q(a, x) by Lentz's continued fraction."""
    if math.isnan(a) or math.isnan(x) or a <= 0.0 or x < 0.0:
        return math.nan
    if x == 0.0:
        return 0.0
    if math.isinf(x):
        return 1.0
    if x >= a + 1.0:
        return 1.0 - _gamma_q_cf(a, x)
    term = s = 1.0 / a
    n = 0
    while abs(term) > _EPS * abs(s):
        n += 1
        if n > _MAX_ITER:
            raise ArithmeticError("incomplete gamma series did not converge (a=%r, x=%r)" % (a, x))
        term *= x / (a + n)
        s += term
    return min(1.0, math.exp(_log_gamma_prefix(a, x)) * s)


def _gamma_q_cf(a, x):
    b = x + 1.0 - a
    c = 1.0 / _TINY
    d = 1.0 / b
    h = d
    i = 0
    while True:
        i += 1
        if i > _MAX_ITER:
            raise ArithmeticError("incomplete gamma fraction did not converge (a=%r, x=%r)" % (a, x))
        an = -i * (i - a)
        b += 2.0
        d = an * d + b
        if abs(d) < _TINY:
            d = _TINY
        c = b + an / c
        if abs(c) < _TINY:
            c = _TINY
        d = 1.0 / d
        de = d * c
        h *= de
        if abs(de - 1.0) <= _EPS:
            return math.exp(_log_gamma_prefix(a, x)) * h


def beta_i(x, y, a, b):
    """regularised incomplete beta I_x(a, b), y = 1 - x.

    Where x <= 0.9 and the largest term of the positive series (_beta_series) comes within its first 100 + 20 sqrt(a),
    that series; else Lentz's continued fraction below (a + 1) / (a + b + 2) and 1 - I_y(b, a) above.  The fraction alone
    is not enough: for b ~ 1e6 and y near 1 its first denominator 1 - (a + b) y / (b + 1) cancels to ~1e-6, and
    1 - I_y(b, a) is off by ~1e-11 where the F test's p-values live.  A longer series would add an ulp per term.  Where the
    fraction is left above the mean, either b is small (a heavy tail, x > 0.9) or (a + b) x exceeds a + 101 + 20 sqrt(a):
    with b large, (a + b) x is close to Gamma(a) distributed and its tail beyond that point is below 1e-40, so the fraction's
    relative error on I_y(b, a) is invisible in 1 - I."""
    if math.isnan(x) or math.isnan(y) or math.isnan(a) or math.isnan(b) or a <= 0.0 or b <= 0.0:
        return math.nan
    if x <= 0.0:
        return 0.0
    if y <= 0.0:
        return 1.0
    peak = ((a + b) * x - (a + 1.0)) / y            # the index of the series' largest term
    if x <= 0.9 and peak <= 100.0 + 20.0 * math.sqrt(a):
        return _beta_series(x, y, a, b)
    if x > (a + 1.0) / (a + b + 2.0):
        return 1.0 - _beta_cf(y, x, b, a)
    return _beta_cf(x, y, a, b)


def _beta_series(x, y, a, b):
    """I_x(a, b) = x^a y^b / (a B(a, b)) sum over n >= 0 of (a + b)_n / (a + 1)_n x^n: every term is positive, so the sum
    keeps a relative error of a few ulps per term; the terms rise to their peak and then fall at least geometrically."""
    t = s = 1.0
    n = 0
    log_scale = 0.0                               # the terms can pass 1e308 before their peak (the prefix is then tiny)
    while True:
        t *= x * ((a + b + n) / (a + 1.0 + n))
        n += 1
        s += t
        if s > 1e250:
            s *= 1e-250
            t *= 1e-250
            log_scale += _LN_1E250
        if t <= 1e-17 * s:
            return min(1.0, math.exp(_log_beta_prefix(x, y, a, b) + log_scale) * s / a)
        if n > _MAX_ITER:
            raise ArithmeticError("incomplete beta series did not converge (x=%r, a=%r, b=%r)" % (x, a, b))


def _beta_cf(x, y, a, b):
    qab, qap, qam = a + b, a + 1.0, a - 1.0
    c = 1.0
    d = 1.0 - qab * x / qap
    if abs(d) < _TINY:
        d = _TINY
    d = 1.0 / d
    h = d
    m = 0
    while True:
        m += 1
        if m > _MAX_ITER:
            raise ArithmeticError("incomplete beta fraction did not converge (x=%r, a=%r, b=%r)" % (x, a, b))
        m2 = 2 * m
        aa = m * (b - m) * x / ((qam + m2) * (a + m2))
        d = 1.0 + aa * d
        if abs(d) < _TINY:
            d = _TINY
        c = 1.0 + aa / c
        if abs(c) < _TINY:
            c = _TINY
        d = 1.0 / d
        h *= d * c
        aa = -(a + m) * (qab + m) * x / ((a + m2) * (qap + m2))
        d = 1.0 + aa * d
        if abs(d) < _TINY:
            d = _TINY
        c = 1.0 + aa / c
        if abs(c) < _TINY:
            c = _TINY
        d = 1.0 / d
        de = d * c
        h *= de
        if abs(de - 1.0) <= _EPS:
            return min(1.0, math.exp(_log_beta_prefix(x, y, a, b)) * h / a)


def chi2_cdf(stat, dof):
    return gamma_p(0.5 * float(dof), 0.5 * float(stat))


def f_cdf(f, d1, d2):
    """the F(d1, d2) distribution's cdf: I_x(d1 / 2, d2 / 2), x = d1 f / (d1 f + d2); +inf gives 1.0."""
    f, d1, d2 = float(f), float(d1), float(d2)
    if math.isnan(f):
        return math.nan
    if f <= 0.0:
        return 0.0
    if math.isinf(f):
        return 1.0
    den = d1 * f + d2
    return beta_i(d1 * f / den, d2 / den, 0.5 * d1, 0.5 * d2)


# ----------------------------------------------------------------------------------- host statistics
class TestResult:
    """p_values [D] f64, dof [D] int64, statistics [D] f64 (host)."""

    def __init__(self, p_values, dof, statistics):
        self.p_values, self.dof, self.statistics = p_values, dof, statistics


def chi_square_from_counts(tables):
    """TestResult from one int64 contingency table [values, labels] per feature."""
    D = len(tables)
    p, dof, st = np.empty(D), np.zeros(D, np.int64), np.empty(D)
    for j, o in enumerate(tables):
        V, L = o.shape
        dof[j] = (V - 1) * (L - 1)
        if dof[j] == 0:
            p[j], st[j] = 1.0, 0.0
            continue
        of = o.astype(np.float64)
        rs, cs = o.sum(1).astype(np.float64), o.sum(0).astype(np.float64)
        n = float(o.sum())
        e = (rs[:, None] * cs[None, :]) / n
        terms = ((of - e) * (of - e) / e).ravel()
        st[j] = np.cumsum(np.concatenate([[0.0], terms]))[-1]
        p[j] = 1.0 - chi2_cdf(st[j], float(dof[j]))
    return TestResult(p, dof, st)


def _seq_sum(rows):
    """rows [G, D] -> [D]: the sum over g in order from +0.0."""
    acc = np.zeros(rows.shape[1])
    for r in rows:
        acc = acc + r
    return acc


def anova_from_totals(sums, counts, ssw_g):
    """TestResult from the class sums [k, D], class counts [k] and centred class sums of squares [k, D]."""
    k = len(counts)
    n = int(counts.sum())
    nf = counts.astype(np.float64)
    means = sums / nf[:, None]
    grand = _seq_sum(sums) / float(n)
    ssw = _seq_sum(ssw_g)
    ssb = _seq_sum(nf[:, None] * ((means - grand) * (means - grand)))
    dfb, dfw = k - 1, n - k
    with np.errstate(invalid="ignore", divide="ignore"):
        f = (ssb / float(dfb)) / (ssw / float(dfw))
    p = np.array([1.0 - f_cdf(v, float(dfb), float(dfw)) for v in f])
    return TestResult(p, np.full(len(f), n - 1, np.int64), f)


def f_value_from_totals(sxx, sxy, syy, n):
    """TestResult from the centred sums of squares sxx [D], cross products sxy [D] and syy."""
    with np.errstate(invalid="ignore", divide="ignore"):
        r = sxy / (np.sqrt(sxx) * math.sqrt(syy))
        f = r * r / (1.0 - r * r) * float(n - 2)
    p = np.array([1.0 - f_cdf(v, 1.0, float(n - 2)) for v in f])
    return TestResult(p, np.full(len(f), n - 2, np.int64), f)


def select(p_values, mode, threshold):
    """the selected feature indices (ascending) under one of Spark's selection modes."""
    p = np.asarray(p_values, np.float64)
    D = len(p)
    order = sorted(range(D), key=lambda j: (math.isnan(p[j]), 0.0 if math.isnan(p[j]) else p[j], j))
    if mode == "numTopFeatures":
        keep = order[:int(threshold)]
    elif mode == "percentile":
        keep = order[:int(D * threshold)]
    elif mode == "fpr":
        keep = [j for j in range(D) if p[j] < threshold]
    elif mode == "fwe":
        keep = [j for j in range(D) if p[j] < threshold / D]
    elif mode == "fdr":
        last = -1
        for i, j in enumerate(order):
            if p[j] <= threshold * (i + 1) / D:
                last = i
        keep = order[:last + 1]
    else:
        raise ValueError("unknown selection mode %r" % (mode,))
    return sorted(keep)


# ----------------------------------------------------------------------------------- device passes
def _check_x(x, what):
    if not (torch.is_tensor(x) and x.is_cuda and x.dim() == 2 and x.dtype == torch.float64):
        raise _lib.B200FlowError("%s needs a CUDA float64 [n, D] matrix" % what)
    if not 1 <= x.shape[1] <= MAX_D:
        raise _lib.UnsupportedParamError("%s supports 1 to %d features, got %d" % (what, MAX_D, x.shape[1]))
    return x.contiguous()


def _check_y(y, n, what):
    if not (torch.is_tensor(y) and y.is_cuda and y.dim() == 1 and y.dtype == torch.float64 and y.shape[0] == n):
        raise _lib.B200FlowError("%s needs a CUDA float64 [n] label" % what)
    return y.contiguous()


def _shards(x, y, row_offset, group, what):
    """Shards of every rank's rows; raises on any rank's non-finite value (an empty shard still joins every collective)."""
    grp = group if group is not None else bdist.group()
    dev = x.device
    if row_offset is None:
        row_offset, _ = bdist.global_offset(x.shape[0], dev, grp)
    sh = bdist.Shards(x.shape[0], row_offset, grp, dev)
    bad = (~torch.isfinite(x)).any().to(torch.int64).reshape(1)
    if y is not None:
        bad = bad + (~torch.isfinite(y)).any().to(torch.int64).reshape(1)
    if grp is not None:
        bdist.all_reduce_(bad, grp)
    if int(bad.item()):
        raise ValueError("%s needs finite features and labels" % what)
    if sh.total == 0:
        raise ValueError("%s needs at least one row" % what)
    return sh


def distinct_tables(x):
    """b200flow_distinct_values on the rows x [n, W]: (tables int64 [W, TABLE_SLOTS] viewed as the keys' bits, counts int32
    [W], overflow int32 [W])."""
    n, W = x.shape
    tables = torch.full((W, TABLE_SLOTS), -1, dtype=torch.int64, device=x.device)
    counts = torch.zeros(W, dtype=torch.int32, device=x.device)
    overflow = torch.zeros(W, dtype=torch.int32, device=x.device)
    call("b200flow_distinct_values", ptr(x), n, W, x.stride(0), ptr(tables), ptr(counts), ptr(overflow))
    return tables, counts, overflow


def dictionaries(x, sh, what):
    """every column's distinct values over every rank's rows: a list of W ascending f64 arrays (host), the same on every
    rank.  Each rank exports its sorted keys in a fixed [W, MAX_CATEGORIES + 2] buffer (keys, +inf padding, overflow flag);
    the union is merged on every rank, and every rank raises if any rank overflowed or a union passes MAX_CATEGORIES."""
    W = x.shape[1]
    tables, _, overflow = distinct_tables(x)
    # the empty slots (a NaN with the sign bit set, which a sort may place first) become +inf, never a key, and sort last
    vals = torch.where(tables == -1, torch.full_like(tables.view(torch.float64), np.inf), tables.view(torch.float64))
    keys = torch.sort(vals, dim=1).values[:, :MAX_CATEGORIES + 1]
    buf = torch.cat([keys, overflow.to(torch.float64).reshape(W, 1)], 1).contiguous()
    parts = [buf] if sh.grp is None else bdist.all_gather_list(buf, sh.grp)
    return merge_dictionaries([p.cpu().numpy() for p in parts], what)


def merge_dictionaries(host, what):
    """the W ascending dictionaries from every rank's exported buffer [W, MAX_CATEGORIES + 2] (host f64: sorted keys,
    +inf padding, overflow flag); raises TooManyValuesError if any rank overflowed a column or its union has more than
    MAX_CATEGORIES values."""
    out = []
    for w in range(host[0].shape[0]):
        v = np.concatenate([h[w, :-1] for h in host])
        u = np.unique(v[np.isfinite(v)])
        if any(h[w, -1] != 0 for h in host) or len(u) > MAX_CATEGORIES:
            raise TooManyValuesError("%s expects factors (categorical values) but found more than %d distinct values in "
                                     "column %d" % (what, MAX_CATEGORIES, w))
        out.append(u)
    return out


def dictionary_ids(values, dict_dev):
    """int32 [n]: the index of each value in the ascending dictionary (device f64), -1 when absent."""
    n = values.shape[0]
    ids = torch.empty(n, dtype=torch.int32, device=values.device)
    call("b200flow_dictionary_ids", ptr(values), n, 1, ptr(dict_dev), int(dict_dev.shape[0]), ptr(ids))
    return ids


def label_dictionary(y, sh, what):
    """(ascending label values (host f64), label ids int32 [n] (device))."""
    d = dictionaries(y.reshape(-1, 1), sh, what + " (label)")[0]
    if len(d) > MAX_LABELS:
        raise _lib.UnsupportedParamError("%s supports at most %d distinct labels, got %d" % (what, MAX_LABELS, len(d)))
    return d, dictionary_ids(y, torch.from_numpy(d).to(y.device))


def contingency_tables(x, label_ids, L, dicts, sh):
    """one int64 table [values, L] (host) per feature, summed over every rank's rows."""
    W = x.shape[1]
    off = np.zeros(W + 1, np.int32)
    off[1:] = np.cumsum([len(d) for d in dicts])
    nv = int(off[-1])
    if nv * L > MAX_CELLS:
        raise _lib.UnsupportedParamError("the contingency tables need %d cells; at most %d are supported" % (nv * L, MAX_CELLS))
    dev = x.device
    counts = torch.zeros(nv * L, dtype=torch.int64, device=dev)
    d_all, off_t = torch.from_numpy(np.concatenate(dicts)).to(dev), torch.from_numpy(off).to(dev)
    call("b200flow_contingency_counts", ptr(x), x.shape[0], W, x.stride(0), ptr(label_ids), L, ptr(d_all), ptr(off_t), nv,
         ptr(counts))
    if sh.grp is not None:
        bdist.all_reduce_(counts, sh.grp)
    host = counts.cpu().numpy().reshape(nv, L)
    return [host[off[w]:off[w + 1]] for w in range(W)]


def chunk_total(x, ids, y, sh, G, width, launch):
    """totals [G, width] f64: launch(rows, ids, y, global row offset, partials [n_chunks, G, width]) over this rank's rows in
    batches of at most PARTIALS_BUDGET bytes of partials, chained in chunk order over every rank (dist.chunk_chain); the same
    bits on every rank."""
    lead, off = sh.lead[sh.rank], sh.offs[sh.rank]
    t0, tail_x, tail_i = bdist.chunk_tail(x, ids, sh)
    tail_y = bdist.chunk_tail(y.reshape(-1, 1), None, sh)[1].reshape(-1) if y is not None else None
    step = max(1, PARTIALS_BUDGET // (8 * G * width)) * bdist.CHUNK
    cut = lambda t, s: t[s:min(s + step, t0)] if t is not None else None          # noqa: E731
    pieces = [(cut(x, s), cut(ids, s), cut(y, s), off + s) for s in range(lead, t0, step)]
    if tail_x.shape[0]:
        pieces.append((tail_x.contiguous(), tail_i, tail_y.contiguous() if y is not None else None, off + t0))

    def run(xs, i_s, ys, go):
        nc = (go + xs.shape[0] - 1) // bdist.CHUNK - go // bdist.CHUNK + 1
        parts = torch.empty((nc, G, width), dtype=torch.float64, device=x.device)
        launch(xs, i_s, ys, go, parts)
        return parts, nc

    if not pieces:
        return bdist.chunk_chain(torch.empty((1, G, width), dtype=torch.float64, device=x.device), 0, G, width, sh)
    first, nc = run(*pieces[0])
    return bdist.chunk_chain(first, nc, G, width, sh, more=(run(*p) for p in pieces[1:]))


def group_sums_total(x, ids, G, sh):
    """(sums [G, W] f64 device, counts int64 [G] host) over every rank's rows: b200flow_group_sums in batches."""
    W = x.shape[1]
    counts = torch.zeros(G, dtype=torch.int64, device=x.device)

    def launch(xs, i_s, _, go, parts):
        call("b200flow_group_sums", ptr(xs), W, ptr(i_s), xs.shape[0], W, G, go, ptr(parts), ptr(counts))

    sums = chunk_total(x, ids, None, sh, G, W, launch)
    if sh.grp is not None:
        bdist.all_reduce_(counts, sh.grp)
    return sums, counts.cpu().numpy()


def centered_moments(xs, ids, G, centers, ys, y_center, row_offset, partials):
    """b200flow_group_centered_moments on the rows xs [n, W] (centers device f64 [G, W]; ys None or device f64 [n])."""
    n, W = xs.shape
    call("b200flow_group_centered_moments", ptr(xs), n, W, xs.stride(0), ptr(ids), G, ptr(centers), ptr(ys),
         float(y_center), row_offset, ptr(partials))


def centered_moments_total(x, ids, G, centers, y, y_center, sh):
    """[G, W] (y None) or [1, 2W + 1] f64 device: the centred sums over every rank's rows in chunk order."""
    W = x.shape[1]
    width = W if y is None else 2 * W + 1

    def launch(xs, i_s, ys, go, parts):
        centered_moments(xs, i_s, G, centers, ys, y_center, go, parts)

    return chunk_total(x, ids if y is None else None, y, sh, G, width, launch)


# ----------------------------------------------------------------------------------- the tests
def chi_square_test(x, y, row_offset=None, group=None):
    """ChiSquareTest of every feature of this rank's rows x [n, D] f64 against the labels y [n] f64 (row_offset = its first
    global row, default from dist.global_offset); identical for any world size.  -> TestResult."""
    x = _check_x(x, "ChiSquareTest")
    y = _check_y(y, x.shape[0], "ChiSquareTest")
    sh = _shards(x, y, row_offset, group, "ChiSquareTest")
    labels, ids = label_dictionary(y, sh, "Chi-square test")
    dicts = dictionaries(x, sh, "Chi-square test")
    return chi_square_from_counts(contingency_tables(x, ids, len(labels), dicts, sh))


def anova_test(x, y, row_offset=None, group=None):
    """ANOVATest of every continuous feature of x [n, D] f64 against the categorical labels y [n] f64.  -> TestResult."""
    x = _check_x(x, "ANOVATest")
    y = _check_y(y, x.shape[0], "ANOVATest")
    sh = _shards(x, y, row_offset, group, "ANOVATest")
    labels, ids = label_dictionary(y, sh, "ANOVA test")
    k = len(labels)
    if k < 2 or sh.total <= k:
        raise ValueError("ANOVATest needs at least two classes and more rows than classes (%d rows, %d classes)" % (sh.total, k))
    sums, counts = group_sums_total(x, ids, k, sh)
    means = sums / torch.from_numpy(counts.astype(np.float64)).to(x.device)[:, None]
    ssw = centered_moments_total(x, ids, k, means.contiguous(), None, 0.0, sh)
    return anova_from_totals(sums.cpu().numpy(), counts, ssw.cpu().numpy())


def f_value_test(x, y, row_offset=None, group=None):
    """FValueTest of every continuous feature of x [n, D] f64 against the continuous label y [n] f64.  -> TestResult."""
    x = _check_x(x, "FValueTest")
    y = _check_y(y, x.shape[0], "FValueTest")
    sh = _shards(x, y, row_offset, group, "FValueTest")
    n = sh.total
    if n <= 2:
        raise ValueError("FValueTest needs more than two rows, got %d" % n)
    mx = group_sums_total(x, None, 1, sh)[0] * (1.0 / n)
    my = float(group_sums_total(y.reshape(-1, 1), None, 1, sh)[0].item()) * (1.0 / n)
    t = centered_moments_total(x, None, 1, mx.contiguous(), y, my, sh).cpu().numpy().reshape(-1)
    D = x.shape[1]
    return f_value_from_totals(t[:D], t[D:2 * D], float(t[2 * D]), n)


def variances(x, row_offset=None, group=None):
    """[D] f64 (host): every feature's unbiased variance, two-pass; 0.0 with a single row."""
    x = _check_x(x, "VarianceThresholdSelector")
    sh = _shards(x, None, row_offset, group, "VarianceThresholdSelector")
    n = sh.total
    mean = group_sums_total(x, None, 1, sh)[0] * (1.0 / n)
    sxx = centered_moments_total(x, None, 1, mean.contiguous(), None, 0.0, sh).cpu().numpy().reshape(-1)
    return sxx / float(n - 1) if n > 1 else np.zeros_like(sxx)
