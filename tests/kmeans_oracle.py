"""numpy restatement of KMeans (k-means|| / random init + Lloyd) and the silhouette of b200flow/kmeans.py (DESIGN.md §5c).

Written from the contract, not from the product: its own Philox, exact squared distances summed in feature order, and the
grouped sum as chunked sequential sums (np.add.accumulate from +0.0 per 4096-row chunk, then over the chunks).  Spark's
loops (initKMeansParallel, LocalKMeans.kMeansPlusPlus, runAlgorithm) are restated as plain loops."""
import numpy as np

CHUNK = 4096
KMNS, KMPP = 0x4B4D4E53, 0x4B4D5050
_M = np.uint64(0xFFFFFFFF)


def philox(seed, purpose, c0, c1, c2, c3):
    """vectorised Philox4x32-10 over uint64 arrays of 32-bit counters -> 4 uint64 arrays of words."""
    k0, k1 = np.uint64((seed & 0xFFFFFFFF) ^ purpose), np.uint64((seed >> 32) & 0xFFFFFFFF)
    c = [np.asarray(v, np.uint64) & _M for v in (c0, c1, c2, c3)]
    c = np.broadcast_arrays(*c)
    c = [v.copy() for v in c]
    for _ in range(10):
        p0 = np.uint64(0xD2511F53) * c[0]
        p1 = np.uint64(0xCD9E8D57) * c[2]
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ k0, p1 & _M, (p0 >> np.uint64(32)) ^ c[3] ^ k1, p0 & _M]
        k0, k1 = (k0 + np.uint64(0x9E3779B9)) & _M, (k1 + np.uint64(0xBB67AE85)) & _M
    return c


def uniforms(w0, w1):
    return ((w0 << np.uint64(21)) | (w1 >> np.uint64(11))).astype(np.float64) * 2.0 ** -53


def row_keys(seed, rows):
    rows = np.asarray(rows, np.uint64)
    w = philox(seed, KMNS, rows, rows >> np.uint64(32), 0, 0)
    return (((w[0] << np.uint64(32)) | w[1]) ^ np.uint64(1 << 63)).view(np.int64)


def select(seed, step, cost, k, sum_cost):
    rows = np.arange(cost.shape[0], dtype=np.uint64)
    w = philox(seed, KMNS, rows, rows >> np.uint64(32), step, 0)
    return uniforms(w[0], w[1]) < ((2.0 * cost) * k) / sum_cost


def sqdist(a, c):
    """[m, D] x [k, D] -> [m, k]: acc = acc + t*t over j in order, t = a_j - c_j."""
    acc = np.zeros((a.shape[0], c.shape[0]))
    for j in range(a.shape[1]):
        t = a[:, j, None] - c[None, :, j]
        acc = acc + t * t
    return acc


def assign(x, centers, block=8192):
    cl = np.empty(x.shape[0], np.int32)
    d = np.empty(x.shape[0])
    for s in range(0, x.shape[0], block):
        dd = sqdist(x[s:s + block], centers)
        cl[s:s + block] = np.argmin(dd, axis=1)                      # the first minimum
        d[s:s + block] = dd[np.arange(dd.shape[0]), cl[s:s + block]]
    return cl, d


def _seq(rows):
    """sequential sum of rows [m, W] in order from +0.0"""
    return np.add.accumulate(np.vstack([np.zeros((1, rows.shape[1])), rows]), axis=0)[-1]


def group_sums(values, ids, G):
    """(totals [G, W], counts [G]) under the chunked rounding contract; global row i = i."""
    values = values.reshape(values.shape[0], -1)
    ids = np.zeros(values.shape[0], np.int64) if ids is None else np.asarray(ids, np.int64)
    W = values.shape[1]
    total = np.zeros((G, W))
    for s in range(0, values.shape[0], CHUNK):
        v, g = values[s:s + CHUNK], ids[s:s + CHUNK]
        part = np.zeros((G, W))
        for gg in np.unique(g):
            part[gg] = _seq(v[g == gg])
        total = total + part                                         # +0.0 partials of absent groups change nothing
    return total, np.bincount(ids, minlength=G)[:G].astype(np.int64)


def distinct_rows(rows):
    out, seen = [], set()
    for r in rows:
        if r.tobytes() not in seen:
            seen.add(r.tobytes())
            out.append(r)
    return np.array(out).reshape(-1, rows.shape[1])


class _Draws:
    def __init__(self, seed):
        self.seed, self.i = seed, 0

    def next(self):
        w = philox(self.seed, KMPP, np.uint64(self.i), np.uint64(self.i >> 32), 0, 0)
        self.i += 1
        return float(uniforms(w[0], w[1]))


def local_kmeans_pp(points, weights, k, seed, max_iter=30):
    """LocalKMeans.kMeansPlusPlus, loop for loop."""
    rnd = _Draws(seed)
    m, D = points.shape

    def pick_weighted():
        total = 0.0
        for w in weights:
            total += w
        r = rnd.next() * total
        i, cur = 0, 0.0
        while i < m and cur < r:
            cur += weights[i]
            i += 1
        return points[max(i - 1, 0)]

    centers = [pick_weighted()]
    cost = sqdist(points, centers[0][None, :])[:, 0]
    for _ in range(1, k):
        s = 0.0
        for c, w in zip(cost, weights):
            s += c * w
        r = rnd.next() * s
        cum, j = 0.0, 0
        while j < m and cum < r:
            cum += weights[j] * cost[j]
            j += 1
        centers.append(points[j - 1] if j > 0 else points[0])
        cost = np.minimum(sqdist(points, centers[-1][None, :])[:, 0], cost)
    centers = np.array(centers)
    old = np.full(m, -1)
    it, moved = 0, True
    while moved and it < max_iter:
        moved = False
        sums, counts = np.zeros((k, D)), np.zeros(k)
        idx = np.argmin(sqdist(points, centers), axis=1)
        for i in range(m):
            sums[idx[i]] = sums[idx[i]] + weights[i] * points[i]
            counts[idx[i]] += weights[i]
            if idx[i] != old[i]:
                moved = True
                old[i] = idx[i]
        for j in range(k):
            if counts[j] == 0.0:
                centers[j] = points[min(int(rnd.next() * m), m - 1)]
            else:
                centers[j] = sums[j] * (1.0 / counts[j])
        it += 1
    return centers


def smallest_key_rows(x, seed, k):
    keys = row_keys(seed, np.arange(x.shape[0]))
    order = np.argsort(keys, kind="stable")[:k]
    return x[order]


def init_parallel(x, k, steps, seed):
    n = x.shape[0]
    cands = [smallest_key_rows(x, seed, 1)]
    new = cands[0]
    cost = np.full(n, np.inf)
    for step in range(1, steps + 1):
        if new.shape[0]:
            cost = np.minimum(cost, assign(x, new)[1])
        sum_cost = group_sums(cost[:, None], None, 1)[0][0, 0]
        new = x[select(seed, step, cost, k, sum_cost)]
        cands.append(new)
    cands = distinct_rows(np.concatenate(cands))
    if cands.shape[0] <= k:
        return cands
    w = np.bincount(assign(x, cands)[0], minlength=cands.shape[0]).astype(np.float64)
    return local_kmeans_pp(cands, w, k, seed)


def lloyd(x, centers, max_iter, tol):
    centers = np.array(centers, np.float64)
    k = centers.shape[0]
    it, converged, cost = 0, False, 0.0
    while it < max_iter and not converged:
        cl, d = assign(x, centers)
        cost = group_sums(d[:, None], None, 1)[0][0, 0]
        sums, counts = group_sums(x, cl, k)
        converged = True
        for j in range(k):
            if counts[j] == 0:
                continue
            c = sums[j] * (1.0 / float(counts[j]))
            if converged and sqdist(c[None, :], centers[j][None, :])[0, 0] > tol * tol:
                converged = False
            centers[j] = c
        it += 1
    cl, _ = assign(x, centers)
    return {"centers": centers, "num_iter": it, "training_cost": float(cost), "cluster_sizes": np.bincount(cl, minlength=k)}


def fit(x, k, init="k-means||", init_steps=2, max_iter=20, tol=1e-4, seed=0):
    if init == "random":
        centers = distinct_rows(smallest_key_rows(x, seed, k))
    else:
        centers = init_parallel(x, k, init_steps, seed)
    return lloyd(x, centers, max_iter, tol)


def silhouette(x, cl):
    cl = np.asarray(cl, np.int64)
    G = int(cl.max()) + 1
    norms = sqdist(x, np.zeros((1, x.shape[1])))[:, 0]
    tot, N = group_sums(np.hstack([x, norms[:, None]]), cl, G)
    Y, psi = tot[:, :-1], tot[:, -1]
    present = np.nonzero(N)[0]
    dot = np.zeros((x.shape[0], G))
    for j in range(x.shape[1]):
        dot = dot + x[:, j, None] * Y[None, :, j]
    Nd = np.where(N > 0, N, 1).astype(np.float64)
    d = (norms[:, None] + psi[None, :] / Nd[None, :]) - (2.0 * dot) / Nd[None, :]
    s = np.zeros(x.shape[0])
    for i in range(x.shape[0]):
        own = cl[i]
        if N[own] <= 1:
            continue
        a = d[i, own] * float(N[own]) / float(N[own] - 1)
        b = min(d[i, g] for g in present if g != own)
        s[i] = 1.0 - a / b if a < b else (b / a - 1.0 if a > b else 0.0)
    return group_sums(s[:, None], None, 1)[0][0, 0] / x.shape[0]
