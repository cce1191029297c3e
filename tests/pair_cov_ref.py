"""numpy statement of cpi_imu_chains_pair_covariance (k_bcr_pair_cov; DESIGN.md section 3q), in any float dtype (float64 or
np.longdouble): the isolated forward phase of the block cyclic reduction, the walk of one pair up its levels, and the sequential
block-Cholesky route that gives every block of one chain's inverse (the extended-precision truth of tests/test_chain_pair_cov.py).

D [n,15,15], E [n-1,15,15] (block (k, k+1)) and cid [n] (the chain of every state) as test_chain_marginals.selinv_ref takes them."""
import numpy as np


def chol(A):
    """Lower Cholesky factors of A [..., 15, 15] in A's dtype (a non-positive pivot gives NaN)."""
    L = np.zeros_like(A)
    with np.errstate(invalid="ignore"):
        for k in range(A.shape[-1]):
            d = np.sqrt(A[..., k, k] - np.sum(L[..., k, :k] ** 2, axis=-1))
            L[..., k, k] = d
            L[..., k + 1:, k] = (A[..., k + 1:, k] - np.einsum("...rq,...q->...r", L[..., k + 1:, :k], L[..., k, :k])) / d[..., None]
    return L


def lsolve(L, B):
    """L^-1 B for lower-triangular L [..., 15, 15] and B [..., 15, c]."""
    X = np.zeros(np.broadcast_shapes(L.shape[:-2], B.shape[:-2]) + B.shape[-2:], dtype=np.result_type(L, B))
    for k in range(L.shape[-1]):
        X[..., k, :] = (B[..., k, :] - np.einsum("...q,...qc->...c", L[..., k, :k], X[..., :k, :])) / L[..., k, k, None]
    return X


def forward(D, E, cid):
    """The forward phase of k_bcr_eliminate_iso / k_bcr_reduce_iso on a zero right-hand side, couplings between chains never read.
    Returns (levels, Sigma_root): level l is (m, stride, Lc, Za, Zb, has_left, has_right) over its odd nodes t (node 2t+1)."""
    D = np.asarray(D)
    dt = D.dtype
    I = np.eye(15, dtype=dt)
    Z = np.zeros((15, 15), dtype=dt)
    Dl, El, stride, m, levels = list(D), list(np.asarray(E, dtype=dt)), 1, len(D), []
    while m > 1:
        c = lambda p: cid[p * stride]
        Lc, Za, Zb, hl, hr = [], [], [], [], []
        for t in range(m // 2):
            i = 2 * t + 1
            L = chol(Dl[i])
            hl.append(c(i - 1) == c(i)); hr.append(i + 1 < m and c(i + 1) == c(i))
            Lc.append(L)
            Za.append(lsolve(L, El[i - 1].T) if hl[-1] else Z)
            Zb.append(lsolve(L, El[i]) if hr[-1] else Z)
        Dn, En = [], []
        for u in range((m + 1) // 2):
            j = 2 * u
            d = Dl[j].copy()
            if j >= 1 and c(j - 1) == c(j):
                d -= Zb[(j - 2) // 2].T @ Zb[(j - 2) // 2]
            if j + 1 < m and c(j + 1) == c(j):
                d -= Za[j // 2].T @ Za[j // 2]
            Dn.append(d)
            if j + 2 < m:
                En.append(-Za[j // 2].T @ Zb[j // 2] if c(j + 2) == c(j) else Z)
        levels.append((m, stride, Lc, Za, Zb, hl, hr))
        Dl, El, stride, m = Dn, En, 2 * stride, (m + 1) // 2
    Li = lsolve(chol(Dl[0]), I)
    return levels, Li.T @ Li


def walk(fw, i, j, drop=None):
    """Sigma_ij by the walk up the levels of fw = forward(...): Sigma_ij = R + sum_{a in A, b in B} C_a Sigma_ab D_b^T from A = {i},
    B = {j}, C = D = I, R = 0.  Each level replaces every node x of A and B it eliminates by its neighbours of x's chain,
    C_nbr += C_x K-/+ with C_x K- = -(C_x Lc^-T) Za, C_x K+ = -(C_x Lc^-T) Zb, after R += (C_x Lc^-T)(D_x Lc^-T)^T where x is in both;
    at the root R += C_0 Sigma_root D_0^T.  Asserts that neither bracket ever holds more than two nodes.  drop(level, x, right):
    a hook that drops the term K+ (right) or K- of node x at a level, for the tests that inject errors."""
    levels, root = fw
    dt = root.dtype
    A, B, R = {i: np.eye(15, dtype=dt)}, {j: np.eye(15, dtype=dt)}, np.zeros((15, 15), dtype=dt)
    for lv, (m, stride, Lc, Za, Zb, hl, hr) in enumerate(levels):
        for x in sorted(set(A) | set(B)):
            if (x // stride) % 2 == 0:
                continue
            t = x // stride // 2
            Y = {id(S): lsolve(Lc[t], S.pop(x).T).T for S in (A, B) if x in S}      # C_x Lc^-T
            if len(Y) == 2:
                R = R + Y[id(A)] @ Y[id(B)].T
            for S in (A, B):
                if id(S) not in Y:
                    continue
                for nb, ok, Zm, right in ((x - stride, hl[t], Za[t], False), (x + stride, hr[t], Zb[t], True)):
                    if ok and not (drop is not None and drop(lv, x, right)):
                        S[nb] = S.get(nb, 0) - Y[id(S)] @ Zm
        assert len(A) <= 2 and len(B) <= 2, (i, j, lv, sorted(A), sorted(B))
        if not A or not B:
            return R
    if A and B:
        R = R + A[0] @ root @ B[0].T
    return R


def sequential(D, E):
    """The sequential route on one chain (D [S,15,15], E [S-1,15,15]) in its dtype: M_k = D_k - U_{k-1}^T U_{k-1} = L_k L_k^T,
    U_k = L_k^-1 E_k, G_k = -L_k^-T U_k (Sigma_{k,j} = G_k Sigma_{k+1,j} for j > k), Sigma_{S-1} = M_{S-1}^-1 and
    Sigma_kk = L_k^-T L_k^-1 + G_k Sigma_{k+1,k+1} G_k^T.  Returns (G [S-1,15,15], Sigma_kk [S,15,15])."""
    S = len(D)
    dt = D.dtype
    I = np.eye(15, dtype=dt)
    Li, G = [], []
    U = None
    for k in range(S):
        M = D[k] - (U.T @ U if U is not None else 0)
        L = chol(M)
        Li.append(lsolve(L, I))
        if k + 1 < S:
            U = lsolve(L, E[k])
            G.append(-Li[-1].T @ U)
    Skk = [None] * S
    Skk[S - 1] = Li[S - 1].T @ Li[S - 1]
    for k in range(S - 2, -1, -1):
        Skk[k] = Li[k].T @ Li[k] + G[k] @ Skk[k + 1] @ G[k].T
    return np.array(G, dtype=dt).reshape(-1, 15, 15), np.array(Skk, dtype=dt)


def sequential_pairs(G, Skk, pairs):
    """Sigma_ij of one chain for local pairs [(i, j)] from sequential()'s G and Sigma_kk: G_i ... G_{j-1} Sigma_jj for i <= j, the
    transpose of (j, i) otherwise."""
    out = []
    for i, j in pairs:
        a, b = min(i, j), max(i, j)
        X = Skk[b]
        for k in range(b - 1, a - 1, -1):
            X = G[k] @ X
        out.append(X if i <= j else X.T)
    return np.array(out, dtype=Skk.dtype).reshape(-1, 15, 15)


def sequential_all(G, Skk):
    """Every block Sigma_ij [S, S, 15, 15] of one chain from sequential()'s G and Sigma_kk."""
    S = len(Skk)
    out = np.zeros((S, S, 15, 15), dtype=Skk.dtype)
    out[np.arange(S), np.arange(S)] = Skk
    for k in range(S - 2, -1, -1):                                 # row k right of the diagonal: G_k (row k+1)
        out[k, k + 1:] = np.einsum("rq,jqc->jrc", G[k], out[k + 1, k + 1:])
    iu = np.triu_indices(S, 1)
    out[iu[1], iu[0]] = out[iu].transpose(0, 2, 1)
    return out
