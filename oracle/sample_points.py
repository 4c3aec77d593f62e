"""TEST INFRASTRUCTURE — NOT PRODUCT CODE.

numpy restatement of kaolin_b200's surface sampling (kaolin_b200/csrc/sample_points.cu), which tests
and benchmarks compare the kernels against:

* ``philox``       Philox4x32-10 (Salmon et al., "Parallel random numbers: as easy as 1, 2, 3", SC 2011)
* ``uniforms``     the random stream: key halves (k0, k1), counter (n, 0, b, j), the word-to-uniform maps
* ``choose``       the float64 CDF of each view (sequential cumsum) and the face choice
* ``face_areas``, ``interpolate``   the reference's rounding (trianglemesh.py:30-40, 76-93), per dtype
* ``sample_points``                  all of the above for dense (B, V, 3) input
* ``grad_*``                         float64 gradients
* ``torch_points``                   the same interpolation in torch, differentiable, at given choices and
                                     uniforms (the DMTet chain test)
"""
import numpy as np

M0, M1, W0, W1 = 0xD2511F53, 0xCD9E8D57, 0x9E3779B9, 0xBB67AE85
_MASK = np.uint64(0xFFFFFFFF)


def philox(c0, c1, c2, c3, k0, k1, rounds=10):
    """Philox4x32 of counters (c0, c1, c2, c3) (uint32 arrays or ints, broadcast) and key (k0, k1)."""
    c = [np.asarray(x, dtype=np.uint64) for x in (c0, c1, c2, c3)]
    c = np.broadcast_arrays(*c)
    c0, c1, c2, c3 = (x.copy() for x in c)
    k0, k1 = np.uint64(k0), np.uint64(k1)
    m0, m1, w0, w1 = np.uint64(M0), np.uint64(M1), np.uint64(W0), np.uint64(W1)
    s32 = np.uint64(32)
    for _ in range(rounds):
        p0, p1 = m0 * c0, m1 * c2          # < 2^64: exact in uint64
        c0, c1, c2, c3 = (p1 >> s32) ^ c1 ^ k0, p1 & _MASK, (p0 >> s32) ^ c3 ^ k1, p0 & _MASK
        k0, k1 = (k0 + w0) & _MASK, (k1 + w1) & _MASK
    return c0, c1, c2, c3


def key_halves(key):
    """(k0, k1): the low and high 32 bits of the int64 key."""
    k = int(np.int64(key)) & 0xFFFFFFFFFFFFFFFF
    return k & 0xFFFFFFFF, k >> 32


def u53(a, b):
    return ((a << np.uint64(21)) | (b >> np.uint64(11))).astype(np.float64) * 2.0 ** -53


def u24(w):
    return (w >> np.uint64(8)).astype(np.float32) * np.float32(2.0 ** -24)


def uniforms(key, B, N, dtype):
    """(r (B, N) float64, u_raw, v (B, N) of dtype) of samples n < N of views b < B."""
    k0, k1 = key_halves(key)
    b = np.arange(B, dtype=np.uint64)[:, None]
    n = np.arange(N, dtype=np.uint64)[None, :]
    w = philox(n, 0, b, 0, k0, k1)
    r = u53(w[0], w[1])
    if np.dtype(dtype) == np.float32:
        return r, u24(w[2]), u24(w[3])
    x = philox(n, 0, b, 1, k0, k1)
    return r, u53(w[2], w[3]), u53(x[0], x[1])


def face_areas(vertices, faces):
    """(B, F) areas of vertices (B, V, 3), each operation rounded in the vertices' dtype."""
    v0, v1, v2 = (vertices[:, faces[:, k]] for k in range(3))
    x, y = v0 - v1, v1 - v2
    a = x[..., 1] * y[..., 2] - x[..., 2] * y[..., 1]
    b = x[..., 2] * y[..., 0] - x[..., 0] * y[..., 2]
    c = x[..., 0] * y[..., 1] - x[..., 1] * y[..., 0]
    return np.sqrt((a * a + b * b) + c * c) * vertices.dtype.type(0.5)


def cdf(areas):
    """The float64 inclusive prefix sum of each view's areas (..., F), in face order."""
    return np.cumsum(np.asarray(areas, dtype=np.float64), axis=-1)


def choose(c, r):
    """The faces of uniforms r (N,) on one view's CDF c (F,): the smallest f with c_f > t, t = r * c_last;
    the first f with c_f = c_last when rounding makes t reach c_last.  Also returns t."""
    last = c[-1]
    t = r * last
    f = np.where(t < last, np.searchsorted(c, t, side="right"), np.searchsorted(c, last, side="left"))
    return f.astype(np.int64), t


def weights(u_raw, v):
    one = u_raw.dtype.type(1)
    u = np.sqrt(u_raw)
    return one - u, u * (one - v), u * v


def interpolate(w, a0, a1, a2):
    """(w0 * a0 + w1 * a1) + w2 * a2 with w (B, N) each and a (B, N, C)."""
    w0, w1, w2 = (x[..., None] for x in w)
    return (w0 * a0 + w1 * a1) + w2 * a2


def sample_points(vertices, faces, num_samples, key, areas=None, face_features=None):
    """-> (points (B, N, 3), choices (B, N) int64, features (B, N, D) or None, (r, u_raw, v), t (B, N))."""
    vertices = np.asarray(vertices)
    B = vertices.shape[0]
    if areas is None:
        areas = face_areas(vertices, faces)
    r, u, v = uniforms(key, B, num_samples, vertices.dtype)
    c = cdf(areas)
    ch = np.empty((B, num_samples), np.int64)
    t = np.empty((B, num_samples), np.float64)
    for b in range(B):
        ch[b], t[b] = choose(c[b], r[b])
    w = weights(u, v)
    bi = np.arange(B)[:, None]
    corners = [vertices[bi, faces[ch, k]] for k in range(3)]
    points = interpolate(w, *corners)
    feats = None
    if face_features is not None:
        feats = interpolate(w, *(face_features[bi, ch, k] for k in range(3)))
    return points, ch, feats, (r, u, v), t


def grad_sample_points(vertices_shape, faces, choices, w, grad_points, face_features_shape=None, grad_features=None):
    """float64 gradients of sample_points: (grad_vertices (B, V, 3), grad_face_features or None)."""
    B = vertices_shape[0]
    gv = np.zeros(vertices_shape, np.float64)
    gp = np.asarray(grad_points, np.float64)
    bi = np.broadcast_to(np.arange(B)[:, None], choices.shape)
    for k in range(3):
        np.add.at(gv, (bi, faces[choices, k]), np.asarray(w[k], np.float64)[..., None] * gp)
    gf = None
    if grad_features is not None:
        gf = np.zeros(face_features_shape, np.float64)
        g = np.asarray(grad_features, np.float64)
        for k in range(3):
            np.add.at(gf, (bi, choices, k), np.asarray(w[k], np.float64)[..., None] * g)
    return gv, gf


def torch_points(vertices, faces, choices, u_raw, v):
    """The interpolation of sample_points in torch at given choices (B, N) and uniforms, with autograd."""
    import torch
    su = torch.sqrt(u_raw)
    w0, w1, w2 = (1 - su)[..., None], (su * (1 - v))[..., None], (su * v)[..., None]
    b = torch.arange(vertices.shape[0], device=vertices.device)[:, None]
    v0, v1, v2 = (vertices[b, faces[choices, k]] for k in range(3))
    return (w0 * v0 + w1 * v1) + w2 * v2


def grad_face_areas(vertices, faces, grad_areas):
    """float64 gradient of face_areas by torch autograd of the same expression (NaN where an area is 0)."""
    import torch
    vt = torch.tensor(np.asarray(vertices, np.float64), requires_grad=True)
    f = torch.as_tensor(faces)
    v0, v1, v2 = vt[:, f[:, 0]], vt[:, f[:, 1]], vt[:, f[:, 2]]
    x, y = v0 - v1, v1 - v2
    a = (x[..., 1] * y[..., 2] - x[..., 2] * y[..., 1]) ** 2
    b = (x[..., 2] * y[..., 0] - x[..., 0] * y[..., 2]) ** 2
    c = (x[..., 0] * y[..., 1] - x[..., 1] * y[..., 0]) ** 2
    (torch.sqrt(a + b + c) * 0.5).backward(torch.tensor(np.asarray(grad_areas, np.float64)))
    return vt.grad.numpy()
