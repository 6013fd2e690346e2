"""numpy fp64 restatement of the MultilayerPerceptronClassifier (DESIGN.md §5d): Spark's flat weight layout, the MLPW
initialisation, forward pass, loss and back-propagation.  Written from the formulas, independently of csrc/mlp.cu."""
import math

import numpy as np

PURPOSE_MLPW = 0x4D4C5057
_M32 = 0xFFFFFFFF


def philox(seed, purpose, c0, c1=0, c2=0, c3=0):
    k0, k1 = (int(seed) & _M32) ^ purpose, (int(seed) >> 32) & _M32
    c = [c0 & _M32, c1 & _M32, c2 & _M32, c3 & _M32]
    for _ in range(10):
        p0, p1 = 0xD2511F53 * c[0], 0xCD9E8D57 * c[2]
        c = [(p1 >> 32) ^ c[1] ^ k0, p1 & _M32, (p0 >> 32) ^ c[3] ^ k1, p0 & _M32]
        k0, k1 = (k0 + 0x9E3779B9) & _M32, (k1 + 0xBB67AE85) & _M32
    return c


def init_weights(layers, seed):
    P = sum((a + 1) * b for a, b in zip(layers[:-1], layers[1:]))
    u = np.empty(P)
    for i in range(P):
        w = philox(seed, PURPOSE_MLPW, i, i >> 32)
        u[i] = float((w[0] << 21) | (w[1] >> 11)) * 2.0 ** -53
    root = np.concatenate([np.full((a + 1) * b, math.sqrt(a)) for a, b in zip(layers[:-1], layers[1:])])
    return (u * 4.8 - 2.4) / root


def unpack(w, layers):
    """[(W [out, in], b [out])] from the flat Spark vector (W column-major, then b)."""
    out, off = [], 0
    for a, b in zip(layers[:-1], layers[1:]):
        W = np.asarray(w[off:off + a * b]).reshape(a, b).T
        out.append((W, np.asarray(w[off + a * b:off + a * b + b])))
        off += (a + 1) * b
    return out


def pack(params):
    return np.concatenate([np.concatenate([W.T.ravel(), b]) for W, b in params])


def forward(w, layers, x):
    """(activations [a_0 = x, a_1, ..., a_{L-1}], logits z)."""
    acts = [np.asarray(x, dtype=np.float64)]
    params = unpack(w, layers)
    for l, (W, b) in enumerate(params):
        z = acts[-1] @ W.T + b
        if l < len(params) - 1:
            acts.append(1.0 / (1.0 + np.exp(-z)))
        else:
            return acts, z


def raw(w, layers, x):
    return forward(w, layers, x)[1]


def softmax(z):
    e = np.exp(z - z.max(1, keepdims=True))
    return e / e.sum(1, keepdims=True)


def loss_grad_sum(w, layers, x, y):
    """(sum over rows of logsumexp(z) - z[y], its gradient in the flat layout)."""
    acts, z = forward(w, layers, x)
    y = np.asarray(y, dtype=np.int64)
    m = z.max(1, keepdims=True)
    lse = m[:, 0] + np.log(np.exp(z - m).sum(1))
    loss = float((lse - z[np.arange(len(y)), y]).sum())
    delta = softmax(z)
    delta[np.arange(len(y)), y] -= 1.0
    params = unpack(w, layers)
    grads = [None] * len(params)
    for l in range(len(params) - 1, -1, -1):
        a = acts[l]
        grads[l] = (delta.T @ a, delta.sum(0))
        if l:
            delta = (delta @ params[l][0]) * a * (1.0 - a)
    return loss, pack(grads)


def loss_grad(w, layers, x, y):
    loss, g = loss_grad_sum(w, layers, x, y)
    return loss / len(y), g / len(y)
