"""GPU (-m gpu): the grid kNN (csrc/knn.cu, the rigidity loss's neighbour sets) at the edges of its search, against
the CUDA brute-force scan and the brute force against a host restatement.

Clouds, each asserting the property it exists for:
  face       tight clusters (sigma 1e-6 .. 1e-4 cell) centred on cell faces computed exactly as the kernel bins a point,
             and points within a few ulps either side of those faces: where the search's stopping bound (the distance
             from the query to its own cell's faces) is least exact;
  clustered  blobs holding hundreds of points per cell, as trained scenes do;
  stacks     exact duplicates (1, 21, 300 copies: clones sit on identical positions) for the index tie-break;
  flat, line, identical, outliers (0.1 % of the points at 1000x the extent);
  tiny       n in {1, 2, k - 1, k, k + 1} for k in {1, 4, 20, 32}.

The brute-force kernel's squared distance, read from `cuobjdump -sass`, is FFMA(dz, dz, FFMA(dx, dx, FMUL(dy, dy)))
(nvcc contracts dx*dx + dy*dy + dz*dz); `d2_host` restates exactly that rounding, so the host check is bit for bit."""
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
F32 = np.float32
KNN_MAX_RES = 160


# ---- the kernel's grid, restated in float32 (knn.cu: grid_res, load_grid, cell_of, the margin) -------------------
def grid_res(n):
    return min(KNN_MAX_RES, max(1, int(math.ceil(np.cbrt(n / 4.0)))))


def grid_params(x):
    """(lo[3], h, inv_h, res) as load_grid forms them: h = fl(fl(max(ext, 1e-20) / res) * 1.0001f), inv_h = fl(1 / h)"""
    lo = x.min(0)
    ext = F32(0)
    for a in range(3):
        ext = max(ext, F32(x[:, a].max() - lo[a]))
    res = grid_res(len(x))
    h = F32(F32(max(ext, F32(1e-20)) / F32(res)) * F32(1.0001))
    return lo, h, F32(F32(1) / h), res


def cell_index(v, lo_a, inv_h, res):
    """cell_of along one axis: trunc(fl(fl(v - lo) * inv_h)), clamped"""
    u = (np.asarray(v, F32) - lo_a).astype(F32) * inv_h
    return np.clip(np.trunc(u.astype(F32)).astype(np.int64), 0, res - 1)


def margin(q, lo, h, inv_h, res):
    """the kernel's distance from each query to its own cell's nearest face: fx = FFMA(-cx, h, fl(q - lo)) per axis
    (contracted: cx * h is not rounded), min(fx, h - fx) over the axes, clamped to [0, h]"""
    m = np.full(len(q), h, F32)
    for a in range(3):
        c = cell_index(q[:, a], lo[a], inv_h, res)
        d = (q[:, a] - lo[a]).astype(F32).astype(np.float64)
        fx = (d - c.astype(np.float64) * np.float64(h)).astype(F32)
        m = np.minimum(m, np.minimum(fx, (h - fx).astype(F32)))
    return np.maximum(m, F32(0))


def face(c, a, lo, h, inv_h, res):
    """the smallest float32 v with cell_index(v) >= c along axis a: the face the kernel's binning puts between cells
    c - 1 and c"""
    v = F32(lo[a] + F32(c) * h)
    while cell_index(v, lo[a], inv_h, res) >= c:
        v = np.nextafter(v, F32(-np.inf), dtype=F32)
    while cell_index(v, lo[a], inv_h, res) < c:
        v = np.nextafter(v, F32(np.inf), dtype=F32)
    return v


# ---- host restatement of the brute force ----------------------------------------------------------------------------
def d2_host(q, p):
    """squared distances [len(q), len(p)] with the kernel's rounding: dx, dy, dz rounded, then
    FFMA(dz, dz, FFMA(dx, dx, dy * dy)); each step is exact in float64 and rounded once to float32"""
    d = [(q[:, None, a] - p[None, :, a]).astype(F32).astype(np.float64) for a in range(3)]
    t = (d[1] * d[1]).astype(F32).astype(np.float64)
    t = (d[0] * d[0] + t).astype(F32).astype(np.float64)
    return (d[2] * d[2] + t).astype(F32)


def knn_host(x, k, chunk=256):
    """(idx, d2) [n, k]: ascending (d2, index), padded with (0, 1e10) like the kernels"""
    n = len(x)
    kk = min(k, n)
    idx = np.zeros((n, k), np.int64)
    d2 = np.full((n, k), F32(1e10), F32)
    for s in range(0, n, chunk):
        d = d2_host(x[s:s + chunk], x)
        thr = np.partition(d, kk - 1, axis=1)[:, kk - 1:kk]
        for r, row in enumerate(d):
            cand = np.nonzero(row <= thr[r])[0]                      # every tie at the k-th distance
            o = cand[np.lexsort((cand, row[cand]))][:kk]             # (d2, index): the lower index among equals
            idx[s + r, :kk], d2[s + r, :kk] = o, row[o]
    return idx, d2


# ---- clouds -----------------------------------------------------------------------------------------------------------
LO, EXT = -0.7, 2.6


def _box(n, rng):
    """n points inside the box [LO, LO + EXT]^3, whose two corners are points 0 and 1 (they fix lo, h and res)"""
    x = (LO + EXT * rng.random((n, 3))).astype(F32)
    x[0], x[1] = F32(LO), F32(LO + EXT)
    return x


def face_cloud(n, seed):
    """uniform background plus clusters of 25..200 points centred on computed cell faces; returns (x, info) with the
    cluster members' indices and the face of each"""
    rng = np.random.default_rng(seed)
    x = _box(n, rng)
    lo, h, inv_h, res = grid_params(x)
    members, faces = [], []
    sig = [1e-6, 1e-5, 1e-4]
    pos = 2
    cells = sorted(set([1, 2, res // 2, res - 2, res - 1]) | set(rng.integers(1, res, 30).tolist()))
    for j in range(max(len(cells), n // 2000)):
        c, a = cells[j % len(cells)], j % 3
        fv = face(c, a, lo, h, inv_h, res)
        m = int(rng.integers(25, 201))
        centre = np.array([F32(lo[b] + (rng.integers(0, res) + 0.5) * h) for b in range(3)], np.float64)
        centre[a] = fv
        pts = centre + sig[j % 3] * float(h) * rng.standard_normal((m, 3))
        pts = pts.astype(F32)
        for t, ul in enumerate(range(-3, 4)):                            # queries within 3 ulps of the face
            v = fv
            for _ in range(abs(ul)):
                v = np.nextafter(v, F32(np.sign(ul) * np.inf), dtype=F32)
            pts[t, a] = v
        if pos + m > n:
            break
        sl = np.arange(pos, pos + m)
        x[sl] = pts
        members.append(sl)
        faces.append((a, fv))
        pos += m
    perm = np.concatenate([[0, 1], 2 + rng.permutation(n - 2)])     # scatter the clusters over the index range
    inv = np.empty(n, np.int64)
    inv[perm] = np.arange(n)
    x = x[perm]
    members = [inv[s] for s in members]
    return x, {"members": members, "faces": faces, "grid": (lo, h, inv_h, res)}


def face_regime(x, info):
    """(points within 1e-5 cell of a computed face, queries whose margin the kernel overestimates: some point in another
    cell is closer than the margin, by the float64 distance)"""
    lo, h, inv_h, res = info["grid"]
    near = unsafe = 0
    for sl, (a, fv) in zip(info["members"], info["faces"]):
        p = x[sl]
        near += int((np.abs(p[:, a].astype(np.float64) - np.float64(fv)) <= 1e-5 * float(h)).sum())
        cells = np.stack([cell_index(p[:, b], lo[b], inv_h, res) for b in range(3)], 1)
        mg = margin(p, lo, h, inv_h, res).astype(np.float64)
        d = np.sqrt(((p[:, None, :].astype(np.float64) - p[None, :, :]) ** 2).sum(-1))
        other = (cells[:, None, :] != cells[None, :, :]).any(-1)
        dmin = np.where(other, d, np.inf).min(1)
        unsafe += int((dmin < mg * math.sqrt(0.9999)).sum())
    return near, unsafe


def clustered_cloud(n, seed):
    """500 Gaussian blobs (sigma 0.4 % of the box) plus 5 % uniform background"""
    rng = np.random.default_rng(seed)
    x = _box(n, rng)
    nb = n - n // 20
    c = LO + 0.1 + (EXT - 0.2) * rng.random((500, 3))
    x[2:2 + nb] = np.clip(c[rng.integers(0, 500, nb)] + 0.01 * rng.standard_normal((nb, 3)), LO, LO + EXT).astype(F32)
    return x


def stack_cloud(n, sizes, seed):
    """a uniform cloud with stacks of identical points (one per size), their members scattered over the indices"""
    rng = np.random.default_rng(seed)
    x = _box(n, rng)
    perm = 2 + rng.permutation(n - 2)
    stacks, pos = [], 0
    for s in sizes:
        members = np.sort(perm[pos:pos + s])
        x[members] = x[members[0]]
        stacks.append(members)
        pos += s
    return x, stacks


def degenerate_cloud(kind, n, seed):
    rng = np.random.default_rng(seed)
    x = _box(n, rng)
    if kind == "flat":
        x[:, 2] = F32(0.25)
    elif kind == "line":
        x[:, 1], x[:, 2] = F32(0.5), F32(-0.125)
    elif kind == "identical":
        x[:] = F32(0.3)
    elif kind == "outliers":
        out = rng.choice(n, max(1, n // 1000), replace=False)
        x[out] = (1000 * EXT * (rng.random((len(out), 3)) - 0.5)).astype(F32)
    return x


# ---- checks -------------------------------------------------------------------------------------------------------------
def _knn(x, k, brute_force):
    from fdgs.knn import knn
    xd = torch.from_numpy(x).to(DEV)[None]
    idx, d2 = knn(xd, xd, k, brute_force=brute_force)
    return idx[0].cpu().numpy(), d2[0].cpu().numpy()


def _check(x, ks, host=None):
    """for each k: grid == brute force bit for bit on indices and distances; with host (default: n <= 20 k) the brute
    force == knn_host bit for bit.  Returns the grid's (idx, d2) of the last k."""
    ks = [ks] if isinstance(ks, int) else list(ks)
    n = len(x)
    hi = hd = None
    if host if host is not None else n <= 20_000:
        hi, hd = knn_host(x, max(ks))
    for k in ks:
        gi, gd = _knn(x, k, False)
        bi, bd = _knn(x, k, True)
        bad = np.nonzero((gi != bi).any(1) | (gd.view(np.uint32) != bd.view(np.uint32)).any(1))[0]
        assert len(bad) == 0, ("grid != brute force", k, len(bad), bad[:5].tolist(), gi[bad[:1]].tolist(), bi[bad[:1]].tolist())
        if hi is not None:
            kk = min(k, n)     # the first min(k, n) of a k_max search are the k search's (the order is total)
            assert np.array_equal(bi[:, :kk], hi[:, :kk]), (k, int((bi[:, :kk] != hi[:, :kk]).any(1).sum()))
            assert np.array_equal(bd[:, :kk].view(np.uint32), hd[:, :kk].view(np.uint32)), (k, int((bd[:, :kk] != hd[:, :kk]).any(1).sum()))
        if n >= k:
            assert (gd[:, 1:] >= gd[:, :-1]).all()
        else:
            assert (gi[:, n:] == 0).all() and (gd[:, n:] == F32(1e10)).all()
    return gi, gd


def test_face_cloud_regime_and_search_small():
    """the face cloud at 8 k points: the regime holds, grid == brute force == host"""
    x, info = face_cloud(8_000, 1)
    near, unsafe = face_regime(x, info)
    assert near >= 500 and unsafe >= 20, (near, unsafe)
    _check(x, (1, 4, 20, 32))


@pytest.mark.parametrize("n", [100_000, 2_000_000])
def test_face_cloud(n):
    """clusters on computed faces: the kernel's shell-0 bound overestimates some queries' distance to the next cell
    (`unsafe`), and the grid must still return the brute force's neighbours"""
    x, info = face_cloud(n, 3)
    near, unsafe = face_regime(x, info)
    assert near >= n // 40 and unsafe >= n // 500, (near, unsafe)
    _check(x, (4, 20, 32) if n <= 100_000 else (20,))


@pytest.mark.parametrize("n", [100_000, 2_000_000])
def test_clustered_cloud(n):
    x = clustered_cloud(n, 5)
    lo, h, inv_h, res = grid_params(x)
    cells = np.stack([cell_index(x[:, a], lo[a], inv_h, res) for a in range(3)], 1)
    _, counts = np.unique((cells[:, 2] * res + cells[:, 1]) * res + cells[:, 0], return_counts=True)
    assert counts.max() >= 200, counts.max()                   # hundreds of points in a cell
    _check(x, 20)


@pytest.mark.parametrize("k", [1, 4, 20, 32])
def test_duplicate_stacks(k):
    """stacks of 1, 21 and 300 identical points: among equal distances the lower index wins, so every member's
    neighbours start with the stack's lowest indices (the point itself only when it is one of them)"""
    x, stacks = stack_cloud(8_000, (1, 21, 300), 2)
    assert all(len(np.unique(x[s], axis=0)) == 1 for s in stacks)
    gi, gd = _check(x, k)
    for s in stacks:
        m = min(k, len(s))
        assert (gi[s, :m] == s[:m][None, :]).all()
        assert (gd[s, :m] == 0).all()
        assert len(s) >= k or (gd[s, len(s)] > 0).all()


@pytest.mark.parametrize("kind", ["flat", "line", "identical", "outliers"])
@pytest.mark.parametrize("k", [1, 20, 32])
def test_degenerate_clouds(kind, k):
    x = degenerate_cloud(kind, 5000 if kind != "identical" else 400, 4)
    lo, h, inv_h, res = grid_params(x)
    ext = [float(x[:, a].max() - x[:, a].min()) for a in range(3)]
    if kind == "flat":
        assert ext[2] == 0 and min(ext[:2]) > 2
    elif kind == "line":
        assert ext[1] == ext[2] == 0 and ext[0] > 2
    elif kind == "identical":
        assert max(ext) == 0 and float(h) < 1e-20
    else:
        assert max(ext) > 500 * EXT
    gi, gd = _check(x, k)
    if kind == "identical":
        assert (gi == np.arange(k)[None, :]).all() and (gd == 0).all()


@pytest.mark.parametrize("k", [1, 4, 20, 32])
def test_tiny_clouds(k):
    rng = np.random.default_rng(k)
    for n in sorted({1, 2, max(1, k - 1), k, k + 1}):
        x = (rng.random((n, 3)) * 2 - 1).astype(F32)
        gi, gd = _check(x, k)
        assert (gi[:, 0] == np.arange(n)).all()


def test_dist_cuda2_on_duplicate_stacks():
    """distCUDA2 (the mean squared distance to the 3 nearest other points) where the k = 4 search returns duplicates with
    lower indices than the point itself, or not the point at all"""
    from fdgs.knn import distCUDA2
    x, stacks = stack_cloud(3000, (2, 3, 4, 5, 21), 6)
    got = distCUDA2(torch.from_numpy(x).to(DEV)).cpu().numpy()
    d = d2_host(x, x).astype(np.float64)
    np.fill_diagonal(d, np.inf)
    best = np.sort(d, axis=1)[:, :3].astype(F32)
    want = (best[:, 0] + best[:, 1] + best[:, 2]) * F32(1.0 / 3.0)     # torch's tensor / 3.0 on CUDA
    assert np.array_equal(got, want), int((got != want).sum())
    for s in stacks:
        if len(s) >= 4:
            assert (got[s] == 0).all()
