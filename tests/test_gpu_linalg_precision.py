"""Matrix.svd / svd_device, Matrix.eigh, Matrix.gemm and Pca.fit on the GPU against references in higher precision than the
kernels': mpmath at 40 digits for matrices up to 64 x 64, f64 LAPACK for f32 inputs, and f64 (or, for f64 GEMM, x87 extended)
products for the large shapes.  Every case asserts which kernel ran, and the shapes sit at the edges where the kernel choice changes
(host twin / device, cluster / warp-per-pair / CTA-per-pair SVD, tensor-core / generic GEMM, K tile edge and split).

The tolerances come from error models, not from observed output:
  * one-sided Jacobi is backward stable column by column, so singular values are within c n eps sigma_max; it stops when every
    pair satisfies |u_p . u_q| <= sqrt(m) eps, so U is orthonormal to a small multiple of sqrt(m) eps; V accumulates ~10 n
    rotations of eps each, so it is orthonormal to 8 n eps;
  * for A = B D with B well conditioned it is also RELATIVELY accurate (Demmel-Veselic): |sigma_i - sigma_i*| <= 2 n eps sigma_i,
    and right vectors within c n eps / relgap_i.  An algorithm that is only absolutely accurate misses both by ~1e10 in f64;
  * eigh's stopping rule is absolute (an off-diagonal entry below eps |A|_F / n is left alone, as the reference's eigen.zig:64-72
    stops on |offdiag|_F <= eps |A|_F), so eigenvalues are asserted to c n eps |A|_2 only, never relatively;
  * a GEMM that accumulates in f64 is within (K + 2) eps_64 (|A||B|)_ij of the exact product before the final rounding to T.
test_error_model_rejects_perturbed_results (no GPU) checks that each bound rejects a result perturbed the way a subtly wrong
kernel would perturb it."""
import contextlib
import functools

import numpy as np
import pytest

import oracle_lib as zo

CLUSTER_CTAS = 8
CLUSTER_SMEM = 200 * 1024     # what one CTA of the SVD cluster may hold (zb_jacobi.cu)
DEVICE_MIN_N = 24             # below this the host entry runs the host twin
WARP_MAX_M = 2048             # the cooperative SVD takes a warp per pair up to this column length, a CTA per pair above


# ---- references -----------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def _mp_svd_cached(key, shape):
    import mpmath
    a = np.frombuffer(key, np.float64).reshape(shape)
    with mpmath.workdps(40):
        _, s, v = mpmath.svd_r(mpmath.matrix(a.tolist()), full_matrices=False, compute_uv=True)
        s = np.array([float(x) for x in s])
        v = np.array([[float(x) for x in v[i, :]] for i in range(v.rows)]).T    # columns = right singular vectors
    order = np.argsort(-s, kind="stable")
    return s[order], v[:, order]


def mp_svd(a):
    """Singular values (descending) and right vectors of the STORED matrix, to 40 digits."""
    a = np.ascontiguousarray(a, np.float64)
    return _mp_svd_cached(a.tobytes(), a.shape)


def ref_singular_values(a):
    """mpmath up to 64 x 64 in f64; f64 LAPACK otherwise (exact for f32 inputs to ~1e-16, far below the f32 bounds)."""
    if a.dtype == np.float64 and a.shape[0] <= 64:
        return mp_svd(a)[0]
    return np.linalg.svd(a.astype(np.float64), compute_uv=False)


def ref_eigenvalues(a):
    if a.dtype == np.float64 and a.shape[0] <= 64:
        import mpmath
        with mpmath.workdps(40):
            e, _ = mpmath.eigsy(mpmath.matrix(a.astype(np.float64).tolist()))
            return np.sort(np.array([float(x) for x in e]))
    return np.linalg.eigvalsh(a.astype(np.float64))


# ---- the error model (plain numpy; the CPU-only test perturbs its inputs) ---------------------------------------------------
def eps_of(dtype):
    return float(np.finfo(dtype).eps)


def assert_sigma_abs(s, ref, eps, c=8):
    """Backward stable: |sigma_i - sigma_i*| <= c n eps sigma_max."""
    s, ref = np.asarray(s, np.float64), np.asarray(ref, np.float64)
    n = ref.size
    assert np.all(np.diff(s) <= 0) and np.all(s >= 0), "singular values not descending / negative"
    err = np.max(np.abs(s - ref)) if n else 0.0
    assert err <= c * n * eps * ref[0], (err / (eps * ref[0]), "eps * sigma_max")


def assert_sigma_rel(s, ref, eps):
    """High relative accuracy: |sigma_i - sigma_i*| <= 2 n eps sigma_i*."""
    s, ref = np.asarray(s, np.float64), np.asarray(ref, np.float64)
    rel = np.max(np.abs(s - ref) / ref)
    assert rel <= 2 * ref.size * eps, (rel / eps, "eps relative")


def assert_orthonormal(q, tol):
    q = np.asarray(q, np.float64)
    err = np.max(np.abs(q.T @ q - np.eye(q.shape[1]))) if q.size else 0.0
    assert err <= tol, (err, tol)


def u_tol(m, eps):
    """|u_p . u_q| <= sqrt(m) eps at convergence, plus the rounding of the f64 dot products and of U to T."""
    return 8 * (np.sqrt(m) + 2) * eps


def assert_u_orthonormal(a, u, s, eps):
    """The stopping rule leaves two kinds of pairs: orthogonal to sqrt(m) eps (u_tol), or skipped as rounding noise because
    |g_p . g_q| <= n eps^2 |A|_F^2 (zb_jacobi.cu, hestenes_rotation), which bounds |u_p . u_q| by that over sigma_p sigma_q.  The
    second term only matters for singular values within a few orders of sqrt(n) eps |A|_F (ill-conditioned or graded A)."""
    m, n = a.shape
    frob2 = float(np.sum(a.astype(np.float64) ** 2))
    s64 = s.astype(np.float64)
    with np.errstate(divide="ignore"):
        skipped = np.where(np.outer(s64, s64) > 0, 2 * n * eps * eps * frob2 / np.outer(s64, s64), np.inf)
    np.fill_diagonal(skipped, 0.0)
    u64 = u.astype(np.float64)
    err = np.abs(u64.T @ u64 - np.eye(n))
    assert np.all(err <= u_tol(m, eps) + skipped), float(np.max(err - skipped))


def v_tol(n, eps):
    return 8 * n * eps


def assert_reconstructs(a, u, s, v, eps):
    """A = U S V^T (or A = U U^T A without V) to 16 n eps sigma_max, elementwise."""
    a64, u64 = a.astype(np.float64), u.astype(np.float64)
    n = a.shape[1]
    smax = float(s[0]) if s.size else 0.0
    rec = u64 @ np.diag(s.astype(np.float64)) @ v.astype(np.float64).T if v is not None else u64 @ (u64.T @ a64)
    err = np.max(np.abs(rec - a64))
    assert err <= 16 * n * eps * smax, (err / (eps * max(smax, 1e-300)), "eps * sigma_max")


def relgaps(ref):
    n = ref.size
    return np.array([min(abs(ref[i] - ref[j]) / (ref[i] + ref[j]) for j in range(n) if j != i) for i in range(n)])


def assert_vectors_rel(v, vref, ref, eps, c):
    """Each right vector within c eps / relgap_i of the reference's, up to sign."""
    v, vref = np.asarray(v, np.float64), np.asarray(vref, np.float64)
    gaps = relgaps(np.asarray(ref, np.float64))
    for i in range(ref.size):
        sign = 1.0 if float(v[:, i] @ vref[:, i]) >= 0 else -1.0
        err = np.linalg.norm(v[:, i] - sign * vref[:, i])
        assert err <= c * eps / gaps[i], (i, err / eps, gaps[i])


def assert_eigenvalues(vals, ref, n, eps, norm2, c=8):
    err = np.max(np.abs(np.asarray(vals, np.float64) - ref))
    assert err <= c * n * eps * norm2, (err / (eps * norm2), "eps * |A|_2")


# ---- device helpers -----------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def zb():
    import torch
    assert torch.cuda.is_available()
    import zignal_b200 as zb
    return zb


def _kernel(zb):
    return zb.lib().zb_last_kernel().decode()


@contextlib.contextmanager
def cluster_off(zb):
    assert zb.lib().zb_tune(b"jacobi.cluster", 0) == 0
    try:
        yield
    finally:
        zb.lib().zb_tune(b"jacobi.cluster", 1)


def cluster_fits(m, n, itemsize, with_v):
    cpc = -(-(n + (n & 1)) // CLUSTER_CTAS)
    return n >= 32 and cpc * (m + (n if with_v else 0)) * itemsize + 16 <= CLUSTER_SMEM


def expected_svd_kernel(m, n, itemsize, with_v, cluster=True):
    if cluster and cluster_fits(m, n, itemsize, with_v):
        return "jacobi_svd_cluster"
    return "jacobi_svd_onesided"      # warp per pair when m <= WARP_MAX_M, a CTA per pair above: one name, one algorithm


def run_svd(zb, a, entry, with_v):
    """-> (u, s, v or None, kernel or None when the host twin ran)."""
    from zignal_b200 import matrix
    launches = zb.lib().zb_kernel_launch_count()
    if entry == "host":
        u, s, v, conv = matrix.svd(a, "skinny_u", with_v)
    else:
        import torch
        ud, sd, vd, conv = matrix.svd_device(torch.from_numpy(np.ascontiguousarray(a)).cuda(), True, with_v)
        u, s, v = ud.cpu().numpy(), sd.cpu().numpy(), (vd.cpu().numpy() if with_v else None)
    assert conv == 0
    assert zb.lib().zb_last_sweeps() <= 20, zb.lib().zb_last_sweeps()     # quadratic convergence, not the sweep limit
    kernel = _kernel(zb) if zb.lib().zb_kernel_launch_count() != launches else None
    return u, s, (v if with_v else None), kernel


def check_svd(a, u, s, v, sref):
    m, n = a.shape
    eps = eps_of(a.dtype)
    assert_sigma_abs(s, sref, eps)
    assert_u_orthonormal(a, u, s, eps)
    if v is not None:
        assert_orthonormal(v, v_tol(n, eps))
    assert_reconstructs(a, u, s, v, eps)


def graded(m, n, dtype, seed):
    rng = np.random.default_rng(seed)
    return (rng.standard_normal((m, n)) @ np.diag(np.logspace(0, -3, n))).astype(dtype)


# ---- 1. SVD kernel paths at their boundaries ---------------------------------------------------------------------------
_BOUNDARY = [(24, 23, True), (24, 24, True), (40, 31, True), (40, 32, True), (45, 33, True), (60, 47, True), (45, 33, False),
             (2048, 40, False), (2049, 40, False)]


@pytest.mark.gpu
@pytest.mark.parametrize("entry", ["host", "device"])
@pytest.mark.parametrize("with_v", [True, False])
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("m,n,cluster", _BOUNDARY)
def test_svd_paths_at_their_boundaries(zb, m, n, cluster, dtype, with_v, entry):
    """n = 23 / 24: host twin, then device (host entry); 31 / 32: warp kernel, then cluster; odd n: the tournament's bye;
    m = 2048 / 2049 with the cluster off: warp per pair, then CTA per pair."""
    a = graded(m, n, dtype, m * 100 + n)
    itemsize = np.dtype(dtype).itemsize
    with (contextlib.nullcontext() if cluster else cluster_off(zb)):
        u, s, v, kernel = run_svd(zb, a, entry, with_v)
    if entry == "host" and n < DEVICE_MIN_N:
        assert kernel is None
    else:
        assert kernel == expected_svd_kernel(m, n, itemsize, with_v, cluster)
    check_svd(a, u, s, v, ref_singular_values(a))
    if kernel is not None and m <= WARP_MAX_M and cluster_fits(m, n, itemsize, with_v):
        # the cluster and the warp-per-pair kernel can both run it: same pair order, same arithmetic -> bit for bit
        with (cluster_off(zb) if cluster else contextlib.nullcontext()):
            u2, s2, v2, k2 = run_svd(zb, a, entry, with_v)
        assert {kernel, k2} == {"jacobi_svd_cluster", "jacobi_svd_onesided"}
        assert np.array_equal(s, s2) and np.array_equal(u, u2) and (v is None or np.array_equal(v, v2))


def _cluster_limit(dtype, with_v, m):
    """The largest n whose problem still fits the cluster's shared memory (m fixed, or m = n when m is None)."""
    itemsize = np.dtype(dtype).itemsize
    n = 32
    while cluster_fits(m or (n + 1), n + 1, itemsize, with_v):
        n += 1
    return n


@pytest.mark.gpu
@pytest.mark.parametrize("entry", ["host", "device"])
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("with_v,m", [(True, 600), (False, None)])
def test_svd_either_side_of_the_cluster_shared_memory_limit(zb, dtype, with_v, m, entry):
    n_lim = _cluster_limit(dtype, with_v, m)
    for n in (n_lim, n_lim + 1):
        rows = m or n
        a = graded(rows, n, dtype, n)
        u, s, v, kernel = run_svd(zb, a, entry, with_v)
        assert kernel == ("jacobi_svd_cluster" if n == n_lim else "jacobi_svd_onesided"), (n, kernel)
        check_svd(a, u, s, v, ref_singular_values(a))
        if n == n_lim:                                    # the warp kernel can run it too: bit for bit
            with cluster_off(zb):
                u2, s2, v2, k2 = run_svd(zb, a, entry, with_v)
            assert k2 == "jacobi_svd_onesided"
            assert np.array_equal(s, s2) and np.array_equal(u, u2) and (v is None or np.array_equal(v, v2))


@functools.lru_cache(maxsize=None)
def _square_case(n, dtype):
    a = graded(n, n, dtype, 7 * n)
    return a, np.linalg.svd(a.astype(np.float64), compute_uv=False)


@pytest.mark.gpu
@pytest.mark.parametrize("with_v", [False, True])
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("n", [512, 1024])
def test_svd_device_large_square(zb, n, dtype, with_v):
    """The sizes Pca.fit reaches through the wgmma covariance (dim 512, 1024): cluster or warp-per-pair kernel by size."""
    a, sref = _square_case(n, dtype)
    u, s, v, kernel = run_svd(zb, a, "device", with_v)
    assert kernel == expected_svd_kernel(n, n, np.dtype(dtype).itemsize, with_v)
    check_svd(a, u, s, v, sref)
    if kernel == "jacobi_svd_cluster":
        with cluster_off(zb):
            u2, s2, v2, k2 = run_svd(zb, a, "device", with_v)
        assert k2 == "jacobi_svd_onesided" and np.array_equal(s, s2) and np.array_equal(u, u2)


# ---- 2. relative accuracy of small singular values ---------------------------------------------------------------------
def _graded_product(dtype):
    """A = B D: B 40 x 32 with kappa(B) = 2.4, D = logspace(0, -10) (f64) or logspace(0, -4) (f32).  The smallest column stays
    far above the noise cut sqrt(n) eps |A|_F, so every sigma is determined to full relative precision by the stored A."""
    rng = np.random.default_rng(11)
    q1, _ = np.linalg.qr(rng.standard_normal((40, 32)))
    q2, _ = np.linalg.qr(rng.standard_normal((32, 32)))
    b = q1 @ np.diag(np.linspace(1.0, 1.0 / 2.4, 32)) @ q2.T
    d = np.logspace(0, -10 if dtype == np.float64 else -4, 32)
    return (b * d).astype(dtype)


@pytest.mark.gpu
@pytest.mark.parametrize("entry", ["host", "device"])
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_svd_small_singular_values_to_high_relative_accuracy(zb, dtype, entry):
    a = _graded_product(dtype)
    eps = eps_of(dtype)
    assert np.sqrt(32) * eps * np.linalg.norm(a.astype(np.float64)) < np.min(np.linalg.norm(a.astype(np.float64), axis=0))
    u, s, v, kernel = run_svd(zb, a, entry, True)
    assert kernel == "jacobi_svd_cluster"
    sref, vref = mp_svd(a)
    assert_sigma_rel(s, sref, eps)
    assert_vectors_rel(v, vref, sref, eps, c=4 * a.shape[1])
    check_svd(a, u, s, v, sref)


# ---- 3. rank deficiency ------------------------------------------------------------------------------------------------
def _deficient(kind, m, dtype):
    """-> (matrix, exact rank)."""
    rng = np.random.default_rng(["zero", "rank1", "rank5", "zero_cols", "dup_cols"].index(kind))
    if kind == "zero":
        return np.zeros((m, 32), dtype), 0
    if kind == "rank1":
        return np.outer(rng.standard_normal(m), rng.standard_normal(32)).astype(dtype), 1
    if kind == "rank5":
        return (rng.standard_normal((m, 5)) @ rng.standard_normal((5, 32))).astype(dtype), 5
    if kind == "zero_cols":
        a = rng.standard_normal((m, 40)).astype(dtype)
        a[:, [0, 17, 39]] = 0
        return a, 37
    assert kind == "dup_cols"
    a = rng.standard_normal((m, 20)).astype(dtype)
    return np.ascontiguousarray(np.concatenate([a, a[:, ::-1]], axis=1)), 20


@pytest.mark.gpu
@pytest.mark.parametrize("path", ["cluster", "warp", "cta"])
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("kind", ["zero", "rank1", "rank5", "zero_cols", "dup_cols"])
def test_svd_rank_deficient(zb, kind, dtype, path):
    """U keeps orthonormal columns when A has a null space: the columns at or below the noise floor sigma_max eps m are completed
    to an orthonormal basis by both entries, and the two entries give the same singular values."""
    m = 2100 if path == "cta" else 48
    a, rank = _deficient(kind, m, dtype)
    n = a.shape[1]
    eps = eps_of(dtype)
    with (contextlib.nullcontext() if path == "cluster" else cluster_off(zb)):
        out = {entry: run_svd(zb, a, entry, True) for entry in ("host", "device")}
    for entry, (u, s, v, kernel) in out.items():
        assert kernel == ("jacobi_svd_cluster" if path == "cluster" else "jacobi_svd_onesided"), (entry, kernel)
        smax = float(s[0])
        assert_orthonormal(u, 200 * m * eps)
        assert_orthonormal(v, v_tol(n, eps))
        assert_reconstructs(a, u, s, v, eps)
        assert np.all(s[rank:].astype(np.float64) <= 4 * n * eps * smax), (entry, s[rank:] / (eps * max(smax, 1e-300)))
        if rank:
            assert_sigma_abs(s, ref_singular_values(a), eps)
        else:
            assert not np.any(s)
    # the same kernel on the same columns; only |g_j| is summed in another order (host loop / device block reduction): two f64
    # sums of m positive terms differ by <= m eps_64 of their value, then both round to T
    s_h, s_d = out["host"][1].astype(np.float64), out["device"][1].astype(np.float64)
    assert np.all(np.abs(s_h - s_d) <= (m * eps_of(np.float64) + eps) * np.maximum(s_h, s_d)), np.max(np.abs(s_h - s_d))


# ---- 4. Pca.fit --------------------------------------------------------------------------------------------------------
def _fit(zb, monkeypatch, data, dtype):
    """Pca.fit, recording the kernel behind each device call it makes."""
    from zignal_b200 import matrix
    from zignal_b200.pca import Pca
    seen = []
    for name in ("gemm_device", "svd_device"):
        def wrapped(*args, _fn=getattr(matrix, name), **kw):
            out = _fn(*args, **kw)
            seen.append(_kernel(zb))
            return out
        monkeypatch.setattr(matrix, name, wrapped)
    p = Pca(dtype)
    p.fit(data)
    return p, seen


def _check_change_of_basis(p, rng, eps, scale):
    """With k = dim the components are a basis: reconstruct(project(v)) == v for ANY v, not only for the training data."""
    dim = p.dim
    for _ in range(4):
        v = (rng.standard_normal(dim) * scale).astype(p.dtype)
        rec = p.reconstruct(p.project(v)).astype(np.float64)
        err = np.max(np.abs(rec - v))
        assert err <= 200 * dim * eps * (np.abs(v).max() + np.abs(p.mean).max()), err


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_pca_fit_grey_image_as_rgb(zb, monkeypatch, dtype):
    """RGB pixels of a grey picture: a rank-1 3 x 3 covariance.  All three components orthonormal, the leading one (1, 1, 1) / sqrt 3
    as the reference computes it, the other two eigenvalues at rounding level."""
    rng = np.random.default_rng(5)
    grey = rng.integers(0, 256, 5000).astype(dtype)
    x = np.ascontiguousarray(np.stack([grey, grey, grey], axis=1))
    eps = eps_of(dtype)
    p, seen = _fit(zb, monkeypatch, x, dtype)
    assert seen == ["gemm_f64" if dtype == np.float64 else "gemm_f32_acc64", "jacobi_svd_onesided"]
    assert p.num_components == 3
    assert_orthonormal(p.components, 200 * 3 * eps)
    _, comps, eig = zo.pca_fit(x)
    assert abs(abs(float(p.components[:, 0].astype(np.float64) @ comps[:, 0].astype(np.float64))) - 1.0) <= 16 * eps
    lam = 3 * np.var(grey.astype(np.float64), ddof=1)
    assert abs(float(p.eigenvalues[0]) - lam) <= 8 * 3 * eps * lam
    assert np.all(np.abs(p.eigenvalues[1:].astype(np.float64)) <= 8 * 3 * eps * lam)
    _check_change_of_basis(p, rng, eps, 100.0)


def _cov64(x):
    import torch
    xd = torch.from_numpy(x).cuda().double()
    xc = xd - xd.mean(0)
    return (xc.T @ xc) / (x.shape[0] - 1)


@pytest.mark.gpu
def test_pca_fit_duplicated_columns_wgmma_and_cluster(zb, monkeypatch):
    """dim 256 with every column present twice (rank 128): the wgmma covariance, then the cluster SVD of a singular matrix."""
    import torch
    rng = np.random.default_rng(9)
    half = (rng.standard_normal((4096, 128)) * np.linspace(3.0, 0.5, 128)).astype(np.float32)
    x = np.ascontiguousarray(np.concatenate([half, half], axis=1))
    eps = eps_of(np.float32)
    p, seen = _fit(zb, monkeypatch, x, np.float32)
    assert seen == ["gemm_xtx_tf32x3_wgmma", "jacobi_svd_cluster"]
    assert p.num_components == 256
    assert_orthonormal(p.components, 200 * 256 * eps)
    ev = torch.linalg.eigvalsh(_cov64(x)).flip(0).cpu().numpy()
    assert np.max(np.abs(p.eigenvalues.astype(np.float64) - ev)) <= 1e-5 * ev[0]
    assert np.all(p.eigenvalues[128:] <= 1e-5 * ev[0])
    _check_change_of_basis(p, rng, eps, 1.0)


@pytest.mark.gpu
@pytest.mark.parametrize("dim,svd_kernel", [(512, "jacobi_svd_cluster"), (1024, "jacobi_svd_onesided")])
def test_pca_fit_large_dim(zb, monkeypatch, dim, svd_kernel):
    """dim 512 / 1024 at n = 8192 f32: eigenvalues within 1e-5 lambda_max of an f64 eigendecomposition of the f64 covariance (the
    3xTF32 covariance is within ~2e-6 max|C|); leading components within 2 * 1e-5 lambda_max / gap (Davis-Kahan) of its vectors."""
    import torch
    rng = np.random.default_rng(dim)
    scale = np.ones(dim)
    scale[:6] = [8.0, 7.0, 6.0, 5.0, 4.0, 3.0]                            # six separated leading eigenvalues over a bulk near 1
    x = (rng.standard_normal((8192, dim)) * scale).astype(np.float32)
    x = np.ascontiguousarray(x @ np.linalg.qr(rng.standard_normal((dim, dim)))[0].astype(np.float32))
    p, seen = _fit(zb, monkeypatch, x, np.float32)
    assert seen == ["gemm_xtx_tf32x3_wgmma", svd_kernel]
    evals, evecs = torch.linalg.eigh(_cov64(x))
    ev, vecs = evals.flip(0).cpu().numpy(), evecs.flip(1).cpu().numpy()
    tol = 1e-5 * ev[0]
    assert np.max(np.abs(p.eigenvalues.astype(np.float64) - ev)) <= tol
    assert_orthonormal(p.components, u_tol(dim, eps_of(np.float32)))
    for i in range(6):
        gap = min(ev[i - 1] - ev[i] if i else np.inf, ev[i] - ev[i + 1])
        c = p.components[:, i].astype(np.float64)
        sin = np.sqrt(max(0.0, 1.0 - float(c @ vecs[:, i]) ** 2))
        assert sin <= 2 * tol / gap, (i, sin, gap)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_pca_fit_gram_path(zb, monkeypatch, dtype):
    """n <= dim: the n x n Gram matrix X X^T / (n - 1) and its cluster SVD; components = X^T u_i / sqrt(lambda_i (n - 1))."""
    import torch
    rng = np.random.default_rng(300)
    n, dim = 300, 1000
    x = rng.standard_normal((n, dim)).astype(dtype)
    eps = eps_of(dtype)
    p, seen = _fit(zb, monkeypatch, x, dtype)
    assert seen == ["gemm_f64" if dtype == np.float64 else "gemm_f32_acc64", "jacobi_svd_cluster"]
    k = p.num_components
    assert k == n - 1
    xd = torch.from_numpy(x).cuda().double()
    xc = xd - xd.mean(0)
    ev = torch.linalg.eigvalsh(xc @ xc.T / (n - 1)).flip(0).cpu().numpy()[:k]
    assert np.max(np.abs(p.eigenvalues.astype(np.float64) - ev)) <= 8 * n * eps * ev[0]
    # comps_i^T comps_j = delta_ij + u_i^T (G - U L U^T) u_j / sqrt(l_i l_j): the Gram SVD's c n eps l_max over l_min
    assert_orthonormal(p.components, 8 * n * eps * ev[0] / ev[k - 1])


# ---- 5. GEMM -----------------------------------------------------------------------------------------------------------
def _f64_xtx(x):
    import torch
    xd = torch.from_numpy(x).cuda().double()
    return (xd.T @ xd).cpu().numpy()


@pytest.mark.gpu
@pytest.mark.parametrize("n", [4096, 4097, 4127])
@pytest.mark.parametrize("dim", [512, 640, 1024])
def test_gemm_xtx_wgmma_ragged_rows(zb, dim, n):
    """X^T X on the tensor cores past dim 384, with a ragged last 32-row chunk (4097) and a ragged last slice (4127)."""
    import torch
    from zignal_b200 import matrix
    rng = np.random.default_rng(dim + n)
    x = rng.standard_normal((n, dim)).astype(np.float32)
    x[-1] *= 5.0                                               # the last row must be counted exactly once
    xd = torch.from_numpy(x).cuda()
    got = matrix.gemm_device(xd, xd, True, False).cpu().numpy()
    assert _kernel(zb) == "gemm_xtx_tf32x3_wgmma"
    exact = _f64_xtx(x)
    assert np.abs(got - exact).max() <= 2e-6 * np.abs(exact).max()
    assert np.array_equal(got, got.T)


@pytest.mark.gpu
def test_gemm_xtx_misaligned_and_aliased_shapes_take_the_generic_kernel(zb):
    """The tensor-core route needs a 16-byte aligned X, and A and B must be the same matrix, not merely the same pointer."""
    import torch
    from zignal_b200 import matrix
    rng = np.random.default_rng(1)
    n, dim = 8192, 256
    buf = torch.from_numpy(rng.standard_normal(n * dim + 1).astype(np.float32)).cuda()
    x = buf[1:].view(n, dim)                                   # storage offset of one float
    assert x.data_ptr() % 16 == 4 and x.is_contiguous()
    got = matrix.gemm_device(x, x, True, False).cpu().numpy()
    assert _kernel(zb) == "gemm_f32_acc64"
    exact = _f64_xtx(x.cpu().numpy())
    assert np.abs(got - exact).max() <= 2e-6 * np.abs(exact).max()
    # one buffer, two shapes: A is n x 256, B its first n * 128 floats read as n x 128; op(A) op(B) is 256 x 128
    a = torch.from_numpy(rng.standard_normal((n, dim)).astype(np.float32)).cuda()
    b = a.view(-1)[:n * 128].view(n, 128)
    assert a.data_ptr() == b.data_ptr()
    got = matrix.gemm_device(a, b, True, False)
    assert _kernel(zb) == "gemm_f32_acc64" and tuple(got.shape) == (dim, 128)
    exact = (a.double().T @ b.double()).cpu().numpy()
    assert np.abs(got.cpu().numpy() - exact).max() <= 2e-6 * np.abs(exact).max()


def _exact_gemm(a, b, ta, tb):
    """op(A) op(B) in x87 extended precision (64-bit significand) and |op(A)| |op(B)|."""
    oa = (a.T if ta else a).astype(np.longdouble)
    ob = (b.T if tb else b).astype(np.longdouble)
    return oa @ ob, np.abs(oa) @ np.abs(ob)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("ta,tb", [(False, False), (True, False), (False, True), (True, True)])
@pytest.mark.parametrize("k", [1, 15, 16, 17, 64, 65, 129, 256, 257, 1000])
def test_gemm_generic_tile_edges_and_k_split(zb, k, ta, tb, dtype):
    """M, N at 63 / 64 / 65 (the 64 x 64 tile), K across the 16-deep slab and the split threshold (K >= 256 splits K across CTAs).
    Elementwise: out = beta C + alpha op(A) op(B) to eps_T (|alpha C*| + |beta C|) + 4 K eps_64 |alpha| (|A||B|)."""
    from zignal_b200 import matrix
    rng = np.random.default_rng(k * 4 + 2 * ta + tb)
    eps, eps64 = eps_of(dtype), eps_of(np.float64)
    alpha, beta = 0.75, -0.5
    for mm in (63, 64, 65):
        for nn in (63, 64, 65):
            a = rng.standard_normal((k, mm) if ta else (mm, k)).astype(dtype)
            b = rng.standard_normal((nn, k) if tb else (k, nn)).astype(dtype)
            c = rng.standard_normal((mm, nn)).astype(dtype)
            got = matrix.gemm(a, b, ta, tb, alpha, beta, c).astype(np.longdouble)
            assert _kernel(zb) == ("gemm_f64" if dtype == np.float64 else "gemm_f32_acc64")
            prod, mag = _exact_gemm(a, b, ta, tb)
            want = beta * c.astype(np.longdouble) + alpha * prod
            bound = 2 * eps * (np.abs(alpha * prod) + np.abs(beta * c.astype(np.longdouble))) + 4 * k * eps64 * alpha * mag
            assert np.all(np.abs(got - want) <= bound), (mm, nn, float(np.max(np.abs(got - want) / bound)))


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("shape", [(65, 33), (4096, 128)])
def test_gemm_alpha_zero_skips_the_product_and_beta_zero_ignores_c(zb, dtype, shape):
    """Matrix.zig:741: alpha == 0 skips op(A) op(B), so NaN in A cannot reach the output (out = beta C exactly); beta == 0
    ignores C, NaN included.  (4096, 128) f32 with A == B is the tensor-core shape."""
    import torch
    from zignal_b200 import matrix
    rng = np.random.default_rng(shape[0])
    x = rng.standard_normal(shape).astype(dtype)
    x[3, 5] = np.nan
    c = rng.standard_normal((shape[1], shape[1])).astype(dtype)
    xd, cd = torch.from_numpy(x).cuda(), torch.from_numpy(c).cuda()
    got = matrix.gemm_device(xd, xd, True, False, 0.0, 0.5, cd).cpu().numpy()
    assert _kernel(zb) == ("gemm_f64" if dtype == np.float64 else "gemm_f32_acc64")
    assert np.array_equal(got, dtype(0.5) * c)
    x[3, 5] = 1.0
    c[0, 0] = np.nan
    exact = x.astype(np.float64).T @ x.astype(np.float64)
    xd, cd = torch.from_numpy(x).cuda(), torch.from_numpy(c).cuda()
    for b in (xd, xd.clone()):                                  # the same matrix (tensor cores when the shape allows) and a copy
        got = matrix.gemm_device(xd, b, True, False, 1.0, 0.0, cd).cpu().numpy()
        assert np.abs(got - exact).max() <= 2e-6 * np.abs(exact).max()      # NaN fails this too


# ---- 6. eigh -----------------------------------------------------------------------------------------------------------
def _symmetric(kind, n, dtype, rng):
    q, _ = np.linalg.qr(rng.standard_normal((n, n)))
    if kind == "random":
        m = rng.standard_normal((n, n))
        a = (m + m.T) / 2
    elif kind == "clustered":                                   # an eigenvalue of multiplicity 8 amid a spread spectrum
        lam = np.concatenate([np.full(8, 1.5), np.linspace(-2.0, 3.0, n - 8)])
        a = q @ np.diag(lam) @ q.T
    elif kind == "indefinite":                                  # alternating signs over three decades
        lam = np.logspace(0, -3, n) * np.where(np.arange(n) % 2, -1.0, 1.0)
        a = q @ np.diag(lam) @ q.T
    elif kind == "rank1":
        x = rng.standard_normal(n)
        a = np.outer(x, x)
    else:
        assert kind == "diagonal"
        a = np.diag(rng.standard_normal(n))
    a = a.astype(dtype)
    return ((a + a.T) * dtype(0.5)).astype(dtype)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("kind", ["random", "clustered", "indefinite", "rank1", "diagonal"])
@pytest.mark.parametrize("n", [23, 24, 255, 256, 257, 512])
def test_eigh_against_extended_precision(zb, n, kind, dtype):
    """Eigenvalues within 8 n eps |A|_2 of mpmath (f64, n <= 64) or f64 LAPACK; V orthonormal to 8 n eps; A V = V L to
    8 n eps |A|_2.  Absolute, not relative: the stopping rule is absolute (module docstring)."""
    from zignal_b200 import matrix
    rng = np.random.default_rng(n * 10 + len(kind))
    a = _symmetric(kind, n, dtype, rng)
    eps = eps_of(dtype)
    launches = zb.lib().zb_kernel_launch_count()
    vals, vecs = matrix.eigh(a)
    if n < DEVICE_MIN_N:
        assert zb.lib().zb_kernel_launch_count() == launches           # the host twin
    else:
        assert _kernel(zb) == "jacobi_eigh_twosided"
    sweeps = zb.lib().zb_last_sweeps()
    if kind != "rank1":                                                # see test_eigh_rank1_stops_before_the_sweep_limit
        assert sweeps <= 20, sweeps
    if kind == "diagonal":                                             # nothing to rotate: 0 sweeps, the diagonal exactly
        assert sweeps == 0
        assert np.array_equal(vals, np.sort(np.diag(a)))
        assert np.array_equal(np.abs(vecs), np.eye(n)[:, np.argsort(np.diag(a), kind="stable")])
        return
    a64 = a.astype(np.float64)
    norm2 = float(np.linalg.norm(a64, 2))
    assert np.all(np.diff(vals) >= 0)
    assert_eigenvalues(vals, ref_eigenvalues(a), n, eps, norm2)
    v64 = vecs.astype(np.float64)
    assert_orthonormal(v64, 8 * n * eps)
    assert np.max(np.abs(a64 @ v64 - v64 * vals.astype(np.float64))) <= 8 * n * eps * norm2


@pytest.mark.gpu
@pytest.mark.xfail(strict=True, reason="known defect: the per-entry threshold eps |A|_F / n is below the rounding noise (~eps lambda) "
                                       "that rotations leave in the row of a rank-1 matrix's one eigenvalue, so eigh rotates noise "
                                       "until the 60-sweep limit; the values and vectors stay within the bounds above")
def test_eigh_rank1_stops_before_the_sweep_limit(zb):
    from zignal_b200 import matrix
    a = _symmetric("rank1", 256, np.float64, np.random.default_rng(0))
    matrix.eigh(a)
    assert _kernel(zb) == "jacobi_eigh_twosided"
    assert zb.lib().zb_last_sweeps() <= 20, zb.lib().zb_last_sweeps()


# ---- the error model rejects what a subtly wrong kernel would return (no GPU) -----------------------------------------------
def test_error_model_rejects_perturbed_results():
    a64 = _graded_product(np.float64)
    sref, vref = mp_svd(a64)
    eps = eps_of(np.float64)
    u = a64 @ vref / sref
    assert_sigma_rel(sref, sref, eps)
    assert_vectors_rel(vref, vref, sref, eps, c=4 * 32)
    assert_orthonormal(u, u_tol(40, eps))
    assert_reconstructs(a64, u, sref, vref, eps)
    # sigma_min off by one part in 1e6: within the absolute bound, outside the relative one
    bad = sref.copy()
    bad[-1] *= 1 + 1e-6
    assert_sigma_abs(bad, sref, eps)
    with pytest.raises(AssertionError):
        assert_sigma_rel(bad, sref, eps)
    # an absolutely accurate algorithm: every sigma off by ~eps sigma_max
    with pytest.raises(AssertionError):
        assert_sigma_rel(sref + 4 * eps * sref[0], sref, eps)
    # the two smallest right vectors rotated into each other by 1e-9 rad (an absolutely accurate vector is off by ~eps / 1e-10)
    t = 1e-9
    vb = vref.copy()
    vb[:, -2], vb[:, -1] = np.cos(t) * vref[:, -2] - np.sin(t) * vref[:, -1], np.sin(t) * vref[:, -2] + np.cos(t) * vref[:, -1]
    with pytest.raises(AssertionError):
        assert_vectors_rel(vb, vref, sref, eps, c=4 * 32)
    # U with a null-space column left at zero, or left as noise / sigma
    ub = u.copy()
    ub[:, -1] = 0
    with pytest.raises(AssertionError):
        assert_orthonormal(ub, 200 * 40 * eps)
    with pytest.raises(AssertionError):
        assert_u_orthonormal(a64, ub, sref, eps)
    ub[:, -1] = u[:, -1] + 1e-6 * u[:, 0]
    with pytest.raises(AssertionError):
        assert_orthonormal(ub, u_tol(40, eps))
    # a reconstruction error of 1e-12 sigma_max
    with pytest.raises(AssertionError):
        assert_reconstructs(a64 + 1e-12 * sref[0] * (np.arange(a64.size).reshape(a64.shape) == 7), u, sref, vref, eps)
    # eigenvalues: one off by 100 n eps |A|
    lam = np.linspace(-1.0, 1.0, 24)
    with pytest.raises(AssertionError):
        assert_eigenvalues(lam + 100 * 24 * eps * (np.arange(24) == 3), lam, 24, eps, 1.0)
