"""float64 oracle of ARIMA(p, d, q) errors by conditional least squares (DESIGN.md section 2 item 16), on top of
``arma_oracle``.

For a gated series (``arma_oracle.hannan_rissanen`` passed its gate): x = (phi, theta), and
  objective  S(x) = sum over C = {s in [p, T): e observed at s} of eps~_s(x)^2, eps~ the forecast recursion of
             ``arma_oracle.recursion`` (zero pre-sample, missing rows filled with their prediction);
  Jacobian   J = d eps~ / dx, exact: on an observed row d u~ = 0 and d eps~ = -d pr, on a missing row d u~ = d pr and
             d eps~ = 0 (``gap_jacobian=False``: the gap-free two-filter form on every row, the control build's rule);
  LM         one pass evaluates S, g = J' eps~, H = J'J at an fp32 point; (H + lam diag H) delta = -g by an in-order
             Cholesky (pivot > PIVOT_TOL x diagonal), x' = fp32(x + delta) must pass the step-down tests, else lam x 10
             with no pass; S(x') < S(x) accepts (lam / 10), otherwise lam x 10; stop 1 converged (an accepted pass lowered
             S by <= RTOL x S), 2 stalled (lam > LAMBDA_MAX), 3 budget (max_iter passes, the first at x0).
Outputs as the library's: the HR row when no step was accepted, otherwise the recursion with the shipped x; sigma =
sqrt(S / |C|) for every gated row.
``lm_replay`` is ``lm`` vectorised over series, with the margin of every discrete decision in units of its float64
noise; the exact-input GPU test replays the kernel with it pass by pass.
"""
from __future__ import annotations

import numpy as np

from ar_oracle import AR_MAX, FP32_EPS, KAPPA_MAX
from arma_oracle import MA_MAX, PIVOT_TOL, _integrate, fit_forecast_arma_packed, recursion, step_down

LAMBDA0 = 1e-3
LAMBDA_MAX = 1e10
RTOL = 1e-6
ITER_DEFAULT = 20
ITER_MAX = 64


def css_eval(e, obs, T: int, p: int, q: int, x, gap_jacobian: bool = True):
    """-> (S, J [T, p + q], eps~ [T], C [T] bool) of one series at x = (phi_1..phi_p, theta_1..theta_q)"""
    x = np.asarray(x, dtype=np.float64)
    phi, th = x[:p], x[p:p + q]
    n = p + q
    u = np.zeros(T + AR_MAX)
    ep = np.zeros(T + MA_MAX)
    du = np.zeros((T + AR_MAX, n))
    de = np.zeros((T + MA_MAX, n))
    J = np.zeros((T, n))
    for s in range(T):
        ul = u[AR_MAX + s - 1 - np.arange(p)] if p else np.zeros(0)
        el = ep[MA_MAX + s - 1 - np.arange(q)] if q else np.zeros(0)
        pr = phi @ ul + th @ el
        dpr = np.concatenate([ul, el])
        if p:
            dpr = dpr + phi @ du[AR_MAX + s - 1 - np.arange(p)]
        if q:
            dpr = dpr + th @ de[MA_MAX + s - 1 - np.arange(q)]
        if obs[s]:
            u[AR_MAX + s] = e[s]
            ep[MA_MAX + s] = e[s] - pr
            de[MA_MAX + s] = -dpr
        else:
            u[AR_MAX + s] = pr
            if gap_jacobian:
                du[AR_MAX + s] = dpr
            else:
                de[MA_MAX + s] = -dpr
        J[s] = de[MA_MAX + s]
    eps = ep[MA_MAX:]
    C = np.asarray(obs[:T], dtype=bool).copy()
    C[:p] = False
    return float(eps[C] @ eps[C]), J, eps, C


def two_filter_jacobian(e, obs, T: int, p: int, q: int, x):
    """J_s = (-v_{s-1..s-p}, -w_{s-1..s-q}), v = (1 + theta(B))^-1 u~, w = (1 + theta(B))^-1 eps~ (exact before the
    first missing row)"""
    x = np.asarray(x, dtype=np.float64)
    th = x[p:p + q]
    _, u, eps = recursion(e, obs, T, x[:p], th, T)
    v, w = np.zeros(T), np.zeros(T)
    for s in range(T):
        v[s] = u[s] - sum(th[k] * v[s - 1 - k] for k in range(q) if s - 1 - k >= 0)
        w[s] = eps[s] - sum(th[k] * w[s - 1 - k] for k in range(q) if s - 1 - k >= 0)
    J = np.zeros((T, p + q))
    for s in range(T):
        for j in range(p):
            J[s, j] = -v[s - 1 - j] if s - 1 - j >= 0 else 0.0
        for k in range(q):
            J[s, p + k] = -w[s - 1 - k] if s - 1 - k >= 0 else 0.0
    return J


def _step(H, g, x, p: int, q: int, lam: float):
    """(trial x' or None, lam) of the step rule: lam x 10 until a pivot-safe, step-down-valid fp32 trial point"""
    n = p + q
    while lam <= LAMBDA_MAX:
        A = H + lam * np.diag(np.diag(H))
        L = np.zeros((n, n))
        ok = True
        for j in range(n):
            dj = A[j, j] - L[j, :j] @ L[j, :j]
            if not dj > PIVOT_TOL * A[j, j]:
                ok = False
                break
            L[j, j] = np.sqrt(dj)
            L[j + 1:, j] = (A[j + 1:, j] - L[j + 1:, :j] @ L[j, :j]) / L[j, j]
        if ok:
            delta = np.linalg.solve(L.T, np.linalg.solve(L, -g))
            xt = (x.astype(np.float64) + delta).astype(np.float32)
            ks = step_down(xt[:p].astype(np.float64)) + step_down(-xt[p:].astype(np.float64))
            if all(abs(k) < KAPPA_MAX for k in ks):
                return xt, lam
        lam *= 10.0
    return None, lam


def lm(e, obs, T: int, p: int, q: int, x0, max_iter: int = 0, gap_jacobian: bool = True):
    """LM of section 2 item 16 from the fp32 point x0 -> dict(x (fp32), S0, S, stop, iters, n_acc, path (S after every
    pass), acc (whether every pass after the first accepted its point), n_C)"""
    max_iter = max_iter or ITER_DEFAULT
    x = np.asarray(x0, dtype=np.float32).copy()
    xt = x
    lam, S, S0, passes, n_acc, stop = LAMBDA0, 0.0, np.nan, 0, 0, 0
    H = g = None
    path, acc = [], []
    n_C = 0
    while True:
        Sn, J, eps, C = css_eval(e, obs, T, p, q, xt, gap_jacobian)
        n_C = int(C.sum())
        passes += 1
        conv = False
        if passes == 1:
            take, S0 = True, Sn
        else:
            take = Sn < S
            conv = take and S - Sn <= RTOL * S
            acc.append(bool(take))
        if take:
            if passes > 1:
                n_acc += 1
                lam /= 10.0
                x = xt
            S = Sn
            H, g = J[C].T @ J[C], J[C].T @ eps[C]
        else:
            lam *= 10.0
        path.append(S)
        if conv:
            stop = 1
        elif lam > LAMBDA_MAX:
            stop = 2
        elif passes >= max_iter:
            stop = 3
        if not stop:
            xt, lam = _step(H, g, x, p, q, lam)
            if xt is None:
                stop = 2
        if stop:
            return dict(x=x, S0=S0, S=S, stop=stop, iters=passes, n_acc=n_acc, path=path, acc=acc, n_C=n_C)


def css_bound(e, obs, T: int, p: int, q: int, x, tau):
    """first-order bound on |S_gpu - S_oracle| at the same x from a per-row error tau of e (the fp32 residuals): eps~
    moves by at most be_s = sum_k |h_k| (tau + sum |phi_j| bu_{s-j}) with h the impulse response of 1 / (1 + theta(z))
    (bu = tau on observed rows, the filled value's bound elsewhere), so |dS| <= sum over C of 2 |eps~_s| be_s + be_s^2,
    plus the float64 rounding of the recursion and the sum; x 2"""
    x = np.asarray(x, dtype=np.float64)
    phi, th = np.abs(x[:p]), np.abs(x[p:p + q])
    _, u, eps = recursion(e, obs, T, x[:p], x[p:p + q], T)
    bu = np.zeros(T + AR_MAX)
    be = np.zeros(T + MA_MAX)
    for s in range(T):
        ar_b = sum(phi[j] * bu[AR_MAX + s - 1 - j] for j in range(p))
        ma_b = sum(th[j] * be[MA_MAX + s - 1 - j] for j in range(q))
        if obs[s]:
            be[MA_MAX + s] = tau + ar_b + ma_b
            bu[AR_MAX + s] = tau
        else:
            bu[AR_MAX + s] = ar_b + ma_b
    be = be[MA_MAX:]
    C = np.asarray(obs[:T], dtype=bool).copy()
    C[:p] = False
    S = float(eps[C] @ eps[C])
    return 2.0 * float(np.sum(2.0 * np.abs(eps[C]) * be[C] + be[C] ** 2)) + 64 * 2.0 ** -52 * T * S


U52 = 2.0 ** -52
MARGINS = ("accept", "conv", "pivot", "kappa", "round")


def s_noise(T: int, S):
    """float64 noise of one evaluation of S over T rows: 64 T 2^-52 S (css_bound's rounding term)"""
    return 64.0 * T * U52 * np.asarray(S, dtype=np.float64)


def h_noise(T: int, k: int) -> float:
    """float64 noise of an entry of H = J'J (of g = J' eps~) relative to sqrt(H_ii H_jj) (to sqrt(H_ii S)), sums in
    another order and the derivative recursion included: 8 (k + sqrt(T)) 2^-52"""
    return 8.0 * (k + np.sqrt(T)) * U52


def rounding_margin(v, err):
    """distance of each float64 v to the nearest fp32 rounding midpoint, in units of err (inf where err is 0)"""
    v = np.asarray(v, dtype=np.float64)
    f = v.astype(np.float32)
    up = f.astype(np.float64) <= v
    nb = np.where(up, np.nextafter(f, np.float32(np.inf)), np.nextafter(f, np.float32(-np.inf)))
    dist = np.abs(v - 0.5 * (f.astype(np.float64) + nb.astype(np.float64)))
    err = np.broadcast_to(np.asarray(err, dtype=np.float64), dist.shape)
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where(err > 0, dist / np.where(err > 0, err, 1.0), np.inf)


def _step_down_batch(a):
    """ar_oracle's step-down test of 1 - sum_j a_j z^j on every row of a [m, k] -> (ok [m], kappa margin [m]): the
    distance of each |kappa| reached to KAPPA_MAX over 64 k 2^-52 / prod (1 - kappa^2) of the stages before it"""
    a = np.array(a, dtype=np.float64)
    m, k = a.shape
    ok, mg, amp = np.ones(m, dtype=bool), np.full(m, np.inf), np.ones(m)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        for j in range(k, 0, -1):
            kap = a[:, j - 1]
            mg = np.where(ok, np.minimum(mg, np.abs(KAPPA_MAX - np.abs(kap)) / (64.0 * k * U52 * amp)), mg)
            ok &= np.abs(kap) < KAPPA_MAX
            den = np.where(ok, 1.0 - kap * kap, 1.0)
            amp = amp / den
            if j > 1:
                a = (a[:, :j - 1] + kap[:, None] * a[:, j - 2::-1]) / den[:, None]
    return ok, mg


def _css_pass(E, OBS, T: int, p: int, q: int, X, gap_jacobian: bool = True):
    """``css_eval`` on every row at once, with [H g; g' S] summed over the rows of C in row order (as the kernel does)
    -> (S [n], g [n, k], H [n, k, k], |C| [n]); X [n, k] the points"""
    n, k = X.shape[0], p + q
    phi, th = X[:, :p], X[:, p:]
    P0 = AR_MAX + 1                                  # history padding: the lag slices never reach index -1
    U, EP = np.zeros((n, T + P0)), np.zeros((n, T + P0))
    DU, DE = np.zeros((n, T + P0, k)), np.zeros((n, T + P0, k))
    S, g, H, nC = np.zeros(n), np.zeros((n, k)), np.zeros((n, k, k)), np.zeros(n, dtype=np.int64)
    for s in range(T):
        i = P0 + s
        ul, el = U[:, i - 1:i - 1 - p:-1], EP[:, i - 1:i - 1 - q:-1]
        pr = np.einsum("nj,nj->n", phi, ul) + np.einsum("nj,nj->n", th, el)
        dpr = np.concatenate([ul, el], axis=1)
        if p:
            dpr = dpr + np.einsum("nj,njk->nk", phi, DU[:, i - 1:i - 1 - p:-1])
        if q:
            dpr = dpr + np.einsum("nj,njk->nk", th, DE[:, i - 1:i - 1 - q:-1])
        o, e = OBS[:, s], E[:, s]
        U[:, i] = np.where(o, e, pr)
        eps = np.where(o, e - pr, 0.0)
        EP[:, i] = eps
        if gap_jacobian:
            DU[:, i] = np.where(o[:, None], 0.0, dpr)
            DE[:, i] = np.where(o[:, None], -dpr, 0.0)
        else:
            DE[:, i] = -dpr
        if s >= p and o.any():
            J = DE[:, i] * o[:, None]
            ec = eps * o
            S += ec * ec
            g += J * ec[:, None]
            H += J[:, :, None] * J[:, None, :]
            nC += o
    return S, g, H, nC


def _step_batch(H, g, S, x, p: int, q: int, lam, T: int):
    """``_step`` on every row at once -> (trial points [m, k] fp32, lam [m], found [m], margins {pivot, kappa, round})

    Margins (in units of the float64 noise of the quantity; below 1 the kernel's float64 may decide otherwise):
      pivot  |d_j - PIVOT_TOL a_jj| over h_noise a_jj max(1, a_jj / |d_j|) (the Schur complement's sensitivity);
      kappa  ``_step_down_batch``;
      round  the distance of x + delta to the nearest fp32 midpoint over the first-order bound on delta's float64
             error, h_noise (|A^-1| w + |delta|) componentwise, w_i = sqrt(a_ii) (sum_k sqrt(a_kk) |delta_k| + sqrt(S)):
             delta' - delta = -A^-1 (dA delta + dg) with |dA_ij| <= h_noise sqrt(a_ii a_jj) (H's entries, Cauchy-Schwarz
             on the row sums, a_ii >= H_ii) and |dg_i| <= h_noise sqrt(a_ii S), plus the rounding of x + delta itself.
             It depends on the row's own system only, so a row is classified the same alone or in any batch."""
    m, k = g.shape
    hn = h_noise(T, k)
    lam = np.array(lam, dtype=np.float64)
    xt = np.zeros((m, k), dtype=np.float32)
    found = np.zeros(m, dtype=bool)
    mg = {key: np.full(m, np.inf) for key in ("pivot", "kappa", "round")}
    eye = np.eye(k)
    while True:
        live = np.flatnonzero(~found & (lam <= LAMBDA_MAX))
        if live.size == 0:
            return xt, lam, found, mg
        Hl = H[live]
        dH = np.diagonal(Hl, axis1=1, axis2=2)
        A = Hl + lam[live, None, None] * (eye * dH[:, None, :])
        L = np.zeros_like(A)
        ok = np.ones(live.size, dtype=bool)
        with np.errstate(divide="ignore", invalid="ignore"):
            for j in range(k):
                ajj = A[:, j, j]
                dj = ajj - np.einsum("nk,nk->n", L[:, j, :j], L[:, j, :j])
                noise = hn * ajj * np.maximum(1.0, ajj / np.abs(dj))
                mp = np.abs(dj - PIVOT_TOL * ajj) / noise
                mg["pivot"][live] = np.minimum(mg["pivot"][live], np.where(ok, mp, np.inf))
                ok &= dj > PIVOT_TOL * ajj
                Ljj = np.sqrt(np.where(ok, dj, 1.0))
                L[:, j, j] = Ljj
                L[:, j + 1:, j] = (A[:, j + 1:, j] - np.einsum("nik,nk->ni", L[:, j + 1:, :j], L[:, j, :j])) / Ljj[:, None]
        good = np.zeros(live.size, dtype=bool)
        if ok.any():
            r = np.flatnonzero(ok)
            Lr = L[r]
            y = np.linalg.solve(Lr, -g[live[r]][:, :, None])
            delta = np.linalg.solve(np.transpose(Lr, (0, 2, 1)), y)[:, :, 0]
            v = x[live[r]].astype(np.float64) + delta
            Ar = A[r]
            Dd = np.sqrt(np.diagonal(Ar, axis1=1, axis2=2))
            # first-order bound: |A^-1| (|dA| |delta| + |dg|), |dA_ij| <= hn sqrt(a_ii a_jj), |dg_i| <= hn sqrt(a_ii S)
            w = Dd * ((Dd * np.abs(delta)).sum(axis=1) + np.sqrt(S[live[r]]))[:, None]
            err = hn * (np.einsum("nij,nj->ni", np.abs(np.linalg.inv(Ar)), w) + np.abs(delta))
            rm = rounding_margin(v, err).min(axis=1)
            mg["round"][live[r]] = np.minimum(mg["round"][live[r]], rm)
            cand = v.astype(np.float32)
            ok_ar, m_ar = _step_down_batch(cand[:, :p].astype(np.float64))
            ok_ma, m_ma = _step_down_batch(-cand[:, p:].astype(np.float64))
            mg["kappa"][live[r]] = np.minimum(mg["kappa"][live[r]], np.minimum(m_ar, m_ma))
            pass_ = ok_ar & ok_ma
            good[r] = pass_
            xt[live[r[pass_]]] = cand[pass_]
        found[live[good]] = True
        lam[live[~good]] *= 10.0


def lm_replay(E, OBS, T: int, p: int, q: int, X0, max_iter: int = 0, gap_jacobian: bool = True, rtol: float = RTOL):
    """``lm`` on every row of E [n, T] / OBS [n, T] from its fp32 point X0 [n, p + q], the rows in lockstep (a row that
    has stopped is left out of later passes), with the smallest margin of every discrete decision on its path ->
    dict(x [n, k] fp32, S0, S, stop, iters, n_acc, n_C [n], acc [n, max_iter] (acc[i, j]: pass j + 2 accepted),
    margin {name: [n]}, ambiguous [n]).

    A margin is the distance of a decision's quantity to its threshold in units of that quantity's float64 noise, the
    difference between two float64 evaluations that sum in another order (the kernel's and this one):
      accept  S_new < S: |S - S_new| / (s_noise(S) + s_noise(S_new)); infinite when the trial point is the accepted one
              bit for bit (S_new is then S exactly on both sides);
      conv    S - S_new <= rtol S: |S - S_new - rtol S| / (s_noise(S) + s_noise(S_new));
      pivot, kappa, round  ``_step_batch``;
      lam     lam > LAMBDA_MAX is decided on a float64 lam that both sides form by the same correctly rounded x 10 and
              / 10 from LAMBDA0, so it has no noise; ``margin["lam"]`` is only the relative distance reached.
    A row is ambiguous when one of accept, conv, pivot, kappa or round falls below 1 on its path."""
    E = np.asarray(E, dtype=np.float64)
    OBS = np.asarray(OBS, dtype=bool)
    n, k = E.shape[0], p + q
    max_iter = max_iter or ITER_DEFAULT
    x = np.array(X0, dtype=np.float32).reshape(n, k)
    xt = x.copy()
    lam, S, S0 = np.full(n, LAMBDA0), np.zeros(n), np.full(n, np.nan)
    H, g = np.zeros((n, k, k)), np.zeros((n, k))
    passes, n_acc, stop, nC = (np.zeros(n, dtype=np.int64) for _ in range(4))
    acc = np.zeros((n, max_iter), dtype=bool)
    margin = {key: np.full(n, np.inf) for key in MARGINS + ("lam",)}
    active = np.ones(n, dtype=bool)
    while active.any():
        idx = np.flatnonzero(active)
        Sn, gn, Hn, nc = _css_pass(E[idx], OBS[idx], T, p, q, xt[idx].astype(np.float64), gap_jacobian)
        nC[idx] = nc
        passes[idx] += 1
        first = passes[idx] == 1
        Sp = S[idx]
        same = (xt[idx].view(np.int32) == x[idx].view(np.int32)).all(axis=1)
        take = first | (Sn < Sp)
        conv = ~first & take & (Sp - Sn <= rtol * Sp)
        with np.errstate(divide="ignore", invalid="ignore"):
            den = s_noise(T, Sp) + s_noise(T, Sn)
            m_acc = np.where(~first & ~same, np.abs(Sp - Sn) / den, np.inf)
            m_conv = np.where(~first & take, np.abs(Sp - Sn - rtol * Sp) / den, np.inf)
        margin["accept"][idx] = np.minimum(margin["accept"][idx], m_acc)
        margin["conv"][idx] = np.minimum(margin["conv"][idx], m_conv)
        S0[idx[first]] = Sn[first]
        a = idx[take & ~first]
        n_acc[a] += 1
        lam[a] /= 10.0
        x[a] = xt[a]
        acc[a, passes[a] - 2] = True
        t = idx[take]
        S[t], H[t], g[t] = Sn[take], Hn[take], gn[take]
        lam[idx[~take]] *= 10.0
        st = np.where(conv, 1, np.where(lam[idx] > LAMBDA_MAX, 2, np.where(passes[idx] >= max_iter, 3, 0)))
        margin["lam"][idx] = np.minimum(margin["lam"][idx], np.abs(lam[idx] / LAMBDA_MAX - 1.0))
        stop[idx] = st
        need = idx[st == 0]
        if need.size:
            xs, lam[need], found, mg = _step_batch(H[need], g[need], S[need], x[need], p, q, lam[need], T)
            for key, v in mg.items():
                margin[key][need] = np.minimum(margin[key][need], v)
            xt[need[found]] = xs[found]
            stop[need[~found]] = 2
        active[idx] = stop[idx] == 0
    amb = np.zeros(n, dtype=bool)
    for key in MARGINS:
        amb |= margin[key] < 1.0
    return dict(x=x, S0=S0, S=S, stop=stop, iters=passes, n_acc=n_acc, n_C=nC, acc=acc, margin=margin, ambiguous=amb)


def fit_forecast_arma_css_packed(y, X, t_fit: int, pred_start: int, n_pred: int, p: int, q: int, d: int = 0,
                                 long_order: int = 0, max_iter: int = 0, gap_jacobian: bool = True, hr=None):
    """``arma_oracle.fit_forecast_arma_packed`` (or ``hr``, its result), then LM on every gated row from fp32 of its
    HR estimate -> that dict with pred / phi / theta / sigma replaced on the refined rows and css_start, css, css_stop,
    iters, refined [n], lm [n] (per-row ``lm`` results, None elsewhere)"""
    res = hr if hr is not None else fit_forecast_arma_packed(y, X, t_fit, pred_start, n_pred, p, q, d, long_order)
    res = dict(res)
    y = np.asarray(y, dtype=np.float64)[:, :t_fit]
    n = len(res["status"])
    T, end = res["T"], pred_start + n_pred
    endz = max(end - d, 0)
    pred, phi, theta, sigma = (np.array(res[k], dtype=np.float64) for k in ("pred", "phi", "theta", "sigma"))
    css_start, css, stop, iters = np.full(n, np.nan), np.full(n, np.nan), np.zeros(n, np.int32), np.zeros(n, np.int32)
    refined = np.zeros(n, dtype=bool)
    lms = [None] * n
    zhat = np.array(res["zhat"], dtype=np.float64)
    for i in np.flatnonzero(res["gated"]):
        x0 = np.r_[res["phi"][i, :p], res["theta"][i, :q]].astype(np.float32)
        r = lm(res["e"][i], res["obs"][i], T, p, q, x0, max_iter, gap_jacobian)
        lms[i] = r
        css_start[i], css[i], stop[i], iters[i] = r["S0"], r["S"], r["stop"], r["iters"]
        sigma[i] = np.sqrt(r["S"] / r["n_C"])
        if r["n_acc"] == 0:
            continue
        refined[i] = True
        x = r["x"].astype(np.float64)
        phi[i] = 0.0
        phi[i, :p] = x[:p]
        theta[i] = 0.0
        theta[i, :q] = x[p:]
        pr, _, _ = recursion(res["e"][i], res["obs"][i], T, x[:p], x[p:], endz)
        zhat[i, d:end] = res["fitted"][i, :endz] + pr
    if refined.any():
        if d == 0:
            pred[refined] = zhat[refined, pred_start:end]
        else:
            yh, _ = _integrate(zhat[refined], y[refined], np.isfinite(y[refined]), t_fit, d, end)
            pred[refined] = yh[:, pred_start:end]
    res.update(pred=pred, phi=phi, theta=theta, sigma=sigma, css_start=css_start, css=css, css_stop=stop, iters=iters,
               refined=refined, lm=lms, zhat=zhat)
    return res


def optimality_gap(e, obs, T: int, p: int, q: int, x):
    """relative decrease of S that SciPy's least_squares finds when started at x: (S(x) - S(x*)) / S(x), with x* kept
    inside the stationary / invertible region by the step-down test (0 when it leaves it)"""
    from scipy.optimize import least_squares

    x = np.asarray(x, dtype=np.float64)
    S0, _, _, C = css_eval(e, obs, T, p, q, x)

    def resid(z):
        _, _, eps, _ = css_eval(e, obs, T, p, q, z)
        return eps[C]

    def jac(z):
        _, J, _, _ = css_eval(e, obs, T, p, q, z)
        return J[C]

    sol = least_squares(resid, x, jac=jac, method="lm", xtol=1e-15, ftol=1e-15, gtol=1e-15, max_nfev=400)
    ks = step_down(sol.x[:p]) + step_down(-sol.x[p:])
    if not all(abs(k) < KAPPA_MAX for k in ks):
        return 0.0
    S1 = float(sol.fun @ sol.fun)
    return max(S0 - S1, 0.0) / S0 if S0 > 0 else 0.0


__all__ = ["LAMBDA0", "LAMBDA_MAX", "RTOL", "ITER_DEFAULT", "ITER_MAX", "FP32_EPS", "css_eval", "two_filter_jacobian",
           "lm", "css_bound", "fit_forecast_arma_css_packed", "optimality_gap", "MARGINS", "s_noise", "h_noise",
           "rounding_margin", "lm_replay"]
