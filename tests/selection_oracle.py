"""numpy restatement of b200flow/selection.py: the dictionaries, the contingency counts, the per-chunk grouped and centred
sums (each a sequential sum in row order from +0.0, as np.cumsum is), their chunk-order totals, and the statistics in the
loop order b200flow/selection.py's docstring states.  The p-values use b200flow.selection's incomplete gamma and beta,
which tests/test_selection.py pins to scipy."""
import numpy as np

from b200flow import selection as bs

CHUNK = 4096


def _seq(v):
    """the sequential sum of v from +0.0."""
    return np.cumsum(np.concatenate([[0.0], np.asarray(v, np.float64)]))[-1]


def dictionary(col):
    """ascending distinct values, -0.0 counted as +0.0."""
    return np.unique(np.where(col == 0.0, 0.0, col))


def contingency(x, y):
    """(label dictionary, one int64 table [values, labels] per feature)."""
    labels = dictionary(y)
    li = np.searchsorted(labels, y)
    out = []
    for j in range(x.shape[1]):
        d = dictionary(x[:, j])
        t = np.zeros((len(d), len(labels)), np.int64)
        np.add.at(t, (np.searchsorted(d, x[:, j]), li), 1)
        out.append(t)
    return labels, out


def chunks(n, row_offset):
    """[(lo, hi)) local row ranges of the 4096-row global chunks rows [0, n) touch."""
    if n == 0:
        return []
    first, last = row_offset // CHUNK, (row_offset + n - 1) // CHUNK
    return [(max(0, c * CHUNK - row_offset), min(n, (c + 1) * CHUNK - row_offset)) for c in range(first, last + 1)]


def group_sum_partials(x, ids, G, row_offset):
    """[n_chunks, G, W]: b200flow_group_sums."""
    out = np.zeros((len(chunks(len(x), row_offset)), G, x.shape[1]))
    for c, (lo, hi) in enumerate(chunks(len(x), row_offset)):
        for g in range(G):
            rows = x[lo:hi][(ids[lo:hi] if ids is not None else np.zeros(hi - lo, int)) == g]
            for w in range(x.shape[1]):
                out[c, g, w] = _seq(rows[:, w])
    return out


def centered_partials(x, ids, G, centers, y, yc, row_offset):
    """[n_chunks, G, W'] of b200flow_group_centered_moments."""
    n, W = x.shape
    cl = chunks(n, row_offset)
    if y is not None:
        out = np.zeros((len(cl), 1, 2 * W + 1))
        for c, (lo, hi) in enumerate(cl):
            dx = x[lo:hi] - centers[0]
            dy = y[lo:hi] - yc
            for w in range(W):
                out[c, 0, w] = _seq(dx[:, w] * dx[:, w])
                out[c, 0, W + w] = _seq(dx[:, w] * dy)
            out[c, 0, 2 * W] = _seq(dy * dy)
        return out
    out = np.zeros((len(cl), G, W))
    for c, (lo, hi) in enumerate(cl):
        g_of = ids[lo:hi] if ids is not None else np.zeros(hi - lo, int)
        for g in range(G):
            d = x[lo:hi][g_of == g] - centers[g]
            for w in range(W):
                out[c, g, w] = _seq(d[:, w] * d[:, w])
    return out


def chain(partials):
    """the chunk-order total of partials [n_chunks, G, W] from +0.0."""
    acc = np.zeros(partials.shape[1:])
    for p in partials:
        acc = acc + p
    return acc


def chi_square(x, y):
    """(p [D], dof [D], statistic [D])."""
    _, tables = contingency(x, y)
    D = len(tables)
    p, dof, st = np.empty(D), np.zeros(D, np.int64), np.empty(D)
    for j, o in enumerate(tables):
        V, L = o.shape
        dof[j] = (V - 1) * (L - 1)
        if dof[j] == 0:
            p[j], st[j] = 1.0, 0.0
            continue
        rs, cs, n = o.sum(1).astype(float), o.sum(0).astype(float), float(o.sum())
        terms = []
        for v in range(V):
            for l in range(L):
                e = (rs[v] * cs[l]) / n
                terms.append((o[v, l] - e) * (o[v, l] - e) / e)
        st[j] = _seq(terms)
        p[j] = 1.0 - bs.chi2_cdf(st[j], float(dof[j]))
    return p, dof, st


def anova(x, y):
    labels = dictionary(y)
    ids = np.searchsorted(labels, y)
    k, n = len(labels), len(y)
    sums = chain(group_sum_partials(x, ids, k, 0))
    cnt = np.bincount(ids, minlength=k)
    means = sums / cnt.astype(float)[:, None]
    ssw_g = chain(centered_partials(x, ids, k, means, None, 0.0, 0))
    grand = chain(sums[:, None, :]).reshape(-1) / float(n)
    ssw = chain(ssw_g[:, None, :]).reshape(-1)
    ssb = chain((cnt.astype(float)[:, None] * ((means - grand) * (means - grand)))[:, None, :]).reshape(-1)
    with np.errstate(invalid="ignore", divide="ignore"):
        f = (ssb / float(k - 1)) / (ssw / float(n - k))
    return np.array([1.0 - bs.f_cdf(v, float(k - 1), float(n - k)) for v in f]), np.full(x.shape[1], n - 1), f


def f_value(x, y):
    n, D = x.shape
    mx = chain(group_sum_partials(x, None, 1, 0))[0] * (1.0 / n)
    my = chain(group_sum_partials(y.reshape(-1, 1), None, 1, 0))[0, 0] * (1.0 / n)
    t = chain(centered_partials(x, None, 1, mx[None, :], y, my, 0))[0]
    with np.errstate(invalid="ignore", divide="ignore"):
        r = t[D:2 * D] / (np.sqrt(t[:D]) * np.sqrt(t[2 * D]))
        f = r * r / (1.0 - r * r) * float(n - 2)
    return np.array([1.0 - bs.f_cdf(v, 1.0, float(n - 2)) for v in f]), np.full(D, n - 2), f


def variances(x):
    n = x.shape[0]
    mean = chain(group_sum_partials(x, None, 1, 0))[0] * (1.0 / n)
    sxx = chain(centered_partials(x, None, 1, mean[None, :], None, 0.0, 0))[0]
    return sxx / float(n - 1) if n > 1 else np.zeros_like(sxx)


def select(p, mode, t):
    """Spark's selection rules, written out separately from b200flow.selection.select."""
    D = len(p)
    key = np.where(np.isnan(p), np.inf, p)
    order = [j for j in np.lexsort((np.arange(D), key, np.isnan(p)))]
    if mode == "numTopFeatures":
        return sorted(order[:int(t)])
    if mode == "percentile":
        return sorted(order[:int(D * t)])
    if mode == "fpr":
        return [j for j in range(D) if p[j] < t]
    if mode == "fwe":
        return [j for j in range(D) if p[j] < t / D]
    ok = [i for i, j in enumerate(order) if p[j] <= t * (i + 1) / D]
    return sorted(order[:ok[-1] + 1]) if ok else []
