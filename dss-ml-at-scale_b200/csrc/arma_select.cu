// arma_select.cu -- (p, d, q) selection by hold-out MSE on levels (DESIGN.md section 2 item 14, section 4.18),
// behind mmf_fit_select_arma_f32.  Per slab and listed d, behind that d's fit (gamma / c hand-off) and
// arima_select_kernel, which scores the q = 0 block of the d and updates the running best:
//   arma_select_kernel  one warp per series; lane c holds candidate c of the call's (p, q >= 1) pairs, q-major:
//     pass A   arma_kernel's pass A and step 1 with the long order m of this d, once for every candidate;
//     pass A2  arma_kernel's u^L and eps^ rings, and the float64 normal equations of every distinct row set
//              R(q, L = max(p, q)): one sequential fma per entry over the rows of R in t order, as arma_kernel,
//              with the entries of all row sets spread over the lanes and kept in shared memory;
//     solve    arma_kernel's in-order Cholesky and step-down tests, one candidate per lane;
//     walk     every gated candidate lane runs its own ARMA recursion from s = 0 and its own level chain in pass
//              B's two fp32 orders (lane-parallel AR part on fully observed chunks, all serial otherwise), and
//              scores the dynamic forecast of the held-out levels;
//     choice   the first minimum over the lanes, compared strictly with the running best;
//     pass B   arma_kernel's, with the winner, only for the rows this launch leads.
// The ring shift and the small helpers come from ar_common.cuh; the blocks it has in common with arma_kernel stay written
// out in each kernel, for the reason arma.cu gives.
#include "ar_common.cuh"

// timing builds only (scripts/bench_arma_select.py --split): 1 ends the kernel after pass A and step 1, 2 after pass A2
// and the solve, 3 after the scoring walk and the choice (no pass B)
#ifndef MMF_ARMASEL_STOP_AFTER
#define MMF_ARMASEL_STOP_AFTER 0
#endif

namespace mmf {
namespace {

constexpr int NR = AR_MAX + MA_MAX;        // regressors of a candidate, at most

// A row set with pmax e lags and q eps^ lags orders its regressors e_{t-1..t-pmax}, eps^_{t-1..t-q}, then the
// target e_t.  Its normal equations are the upper triangle, column-major, without the target's own square.  Source
// code of a regressor: k for e_{t-k} (0: the target), 16 + k for eps^_{t-k}.
__device__ __forceinline__ uint32_t reg_src(int x, int pmax, int q) {
  return x < pmax ? (uint32_t)(x + 1) : (x < pmax + q ? 16u + (uint32_t)(x - pmax + 1) : 0u);
}
__device__ __forceinline__ const double* src_base(const double* sE, const double* sV, uint32_t code) {
  return (code & 16u ? sV : sE) + 32 - (int)(code & 15u);
}

// d.t_fit: fit rows of a.y (z' for d >= 1); ma: the levels (ma.d = 0: ma.y is a.y); ar: staging and the phi / order /
// sigma outputs; sel: this d's arima_select_kernel arguments (its running best, n_hold, the orders)
__global__ void __launch_bounds__(THREADS, 2)
arma_select_kernel(const DesignView d, const FitArgs a, const ArArgs ar, const ArimaArgs ma, const ArimaSelArgs sel,
                   const ArmaSelArgs hs) {
  __shared__ float4 s_a[4][TC];
  __shared__ uint32_t s_nz[TC];
  __shared__ double s_e[WARPS][64];        // residuals e of the previous and the current 32 rows (0 where missing)
  __shared__ double s_u[WARPS][64];        // filled long-AR residuals u^L, same rows
  __shared__ double s_v[WARPS][64];        // innovation estimates eps^, same rows (0 where missing)
  __shared__ double s_psi[WARPS][32];      // psi_1..psi_32
  __shared__ uint32_t s_rm[WARPS][32];     // rows of the current chunk in each row set
  extern __shared__ double s_dyn[];        // [WARPS][n_ent] normal-equation entries, then [n_ent] entry codes
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * WARPS + warp;
  const bool live = row < a.n;
  const int m = hs.m;
  const int dd = ma.d;
  const int T = d.t_fit;                   // fit rows of a.y
  const int TL = ma.t_fit;                 // level fit rows
  const int end = a.pred_start + a.n_pred; // level rows [pred_start, end)
  const int endz = end - dd;
  const bool first = sel.d_index == 0;
  const int n_ent = hs.n_ent;
  double* __restrict__ sE = s_e[warp];
  double* __restrict__ sU = s_u[warp];
  double* __restrict__ sV = s_v[warp];
  double* __restrict__ sG = s_dyn + warp * n_ent;
  uint32_t* __restrict__ s_code = reinterpret_cast<uint32_t*>(s_dyn + WARPS * n_ent);

  int st = MMF_STATUS_EMPTY;
  float g[P], c = 0.f;
#pragma unroll
  for (int k = 0; k < P; ++k) g[k] = 0.f;
  ArimaSelBest rb{0.0, -1, -1, 0};         // the running best, this d's q = 0 block included
  if (live) {
    st = a.status[row];
    const float4* gp = reinterpret_cast<const float4*>(a.out_gamma + row * P);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float4 v = gp[k];
      g[4 * k] = v.x; g[4 * k + 1] = v.y; g[4 * k + 2] = v.z; g[4 * k + 3] = v.w;
    }
    c = a.out_c[row];
    rb = sel.best[row];
  }
  const bool work = live && st != MMF_STATUS_EMPTY && hs.n_pq > 0;
  const float* __restrict__ zr = a.y + (live ? row : 0) * a.ld_y;
  const float* __restrict__ yr = ma.y + (live ? row : 0) * ma.ld_y;
  const bool q0_lead = rb.d == dd;         // arima_select_kernel of this d took the lead: the leader has q = 0

  // the entry codes: entry e of row set r at index j (j + 1) / 2 + i is (r, regressor i, regressor j)
  for (int e = threadIdx.x; e < n_ent; e += THREADS) {
    int r = 0;
    while (r + 1 < hs.n_rs && hs.rs_off[r + 1] <= e) ++r;
    const int idx = e - hs.rs_off[r];
    int j = 0;
    while ((j + 1) * (j + 2) / 2 <= idx) ++j;
    const int i = idx - j * (j + 1) / 2;
    const int pm = hs.rs_pmax[r], qq = hs.rs_q[r];
    s_code[e] = (uint32_t)r | reg_src(i, pm, qq) << 8 | reg_src(j, pm, qq) << 16;
  }

  // this lane's candidate (lanes >= n_pq repeat the last one and never take part)
  const bool cand = lane < hs.n_pq;
  const int ci = min(lane, max(hs.n_pq - 1, 0));
  const int p = hs.pq_p[ci], q = hs.pq_q[ci], rs = hs.pq_rs[ci];
  const int nreg = p + q;
  const int pmax = hs.rs_pmax[rs], off = hs.rs_off[rs];

  // ---- pass A: residuals, n_obs, used columns and r_0 (own lane), r_{lane+1} (lane k sums lag k + 1)
  sE[lane] = 0.0;
  double acc0 = 0.0, accl = 0.0;
  int n_obs = 0;
  uint32_t colmask = 0u;
  if (__syncthreads_or(work)) {
    for (int c0 = 0; c0 < T; c0 += TC) {
      stage(s_a, s_nz, d, ar, c0);
      __syncthreads();
      if (work) {
#pragma unroll 1
        for (int t0 = c0; t0 < min(c0 + TC, T); t0 += 32) {
          const int t = t0 + lane;
          const float yv = t < T ? __ldg(zr + t) : 0.f;
          const bool obs = t < T && finite_f(yv);
          const float e = obs ? yv - fitted(s_a, t - c0, g, c) : 0.f;
          n_obs += __popc(__ballot_sync(0xffffffffu, obs));
          colmask |= obs ? s_nz[t - c0] : 0u;
          acc0 = fma((double)e, (double)e, acc0);
          const double ed = (double)e;
          sE[32 + lane] = ed;
          __syncwarp();
          if (lane < m) {
#pragma unroll 8
            for (int j = 0; j < 32; ++j) accl = fma(sE[32 + j], sE[31 + j - lane], accl);
          }
          __syncwarp();
          sE[lane] = ed;
          __syncwarp();
        }
      }
      __syncthreads();
    }
  }

  // ---- step 1: Levinson-Durbin to order m with the kappa stop; lane i holds psi_{i+1} and r_{i+1}
  acc0 = warp_sum(acc0);
  colmask = __reduce_or_sync(0xffffffffu, colmask);
  uint32_t used = d.kept_mask & colmask;
  if (st == MMF_STATUS_RANKDEF) {
#pragma unroll
    for (int k = 0; k < P; ++k) used &= g[k] != 0.f ? ~0u : ~(1u << k);
  }
  const int k_used = __popc(used);
  double psi = 0.0;
  int m_i = 0;
  if (work) {
    const double inv = 1.0 / (double)max(n_obs, 1);
    const double r0 = acc0 * inv, rl = accl * inv;
    double var = r0;
    bool go = n_obs - k_used > m && r0 > 0.0;
    for (int j = 1; j <= m && go; ++j) {
      const double rr = __shfl_sync(0xffffffffu, rl, (j - lane - 2) & 31);     // r_{j - (lane + 1)}
      const double num = __shfl_sync(0xffffffffu, rl, j - 1) - warp_sum(lane + 1 < j ? psi * rr : 0.0);
      const double kap = num / var;
      if (fabs(kap) >= (double)MMF_AR_KAPPA_MAX) {
        go = false;
      } else {
        const double mirror = __shfl_sync(0xffffffffu, psi, (j - lane - 2) & 31);  // psi_{j - (lane + 1)}
        psi = lane + 1 < j ? psi - kap * mirror : (lane + 1 == j ? kap : psi);
        var *= 1.0 - kap * kap;
        m_i = j;
      }
    }
  }
  s_psi[warp][lane] = psi;

#if MMF_ARMASEL_STOP_AFTER == 1
  return;                                  // timing build: pass A and step 1 only
#endif
  // ---- pass A2: u^L, eps^, and the normal equations of every row set (lane owns entries lane, lane + 32, ..; lane r
  // counts the rows of row set r)
  const bool hr_ok = work && m_i >= 1;
  for (int e = lane; e < n_ent; e += 32) sG[e] = 0.0;
  int n_R = 0;
  sE[lane] = 0.0; sU[lane] = 0.0; sV[lane] = 0.0;
  __syncwarp();
  const int rs_L = lane < hs.n_rs ? hs.rs_L[lane] : 0;
  const int rs_lo = lane < hs.n_rs ? m + hs.rs_q[lane] : INT32_MAX;   // first row of row set `lane`
  uint32_t bprev = 0u;
  if (__syncthreads_or(hr_ok)) {
    for (int c0 = 0; c0 < T; c0 += TC) {
      stage(s_a, s_nz, d, ar, c0);
      __syncthreads();
      if (hr_ok) {
#pragma unroll 1
        for (int t0 = c0; t0 < min(c0 + TC, T); t0 += 32) {
          const int t = t0 + lane;
          const float yv = t < T ? __ldg(zr + t) : 0.f;
          const bool obs = t < T && finite_f(yv);
          const float e = obs ? yv - fitted(s_a, t - c0, g, c) : 0.f;
          const uint32_t bal = __ballot_sync(0xffffffffu, obs);
          const double ed = (double)e;
          sE[32 + lane] = ed;
          sU[32 + lane] = ed;
          __syncwarp();
          // missing fit rows of the chunk, in order: u^L_s = sum_k psi_k u^L_{s-k}
          uint32_t miss = ~bal;
          if (T - t0 < 32) miss &= (1u << (T - t0)) - 1u;
          while (miss) {
            const int j = __ffs(miss) - 1;
            miss &= miss - 1u;
            const double v = warp_sum(lane < m_i ? psi * sU[31 + j - lane] : 0.0);
            if (lane == 0) sU[32 + j] = v;
            __syncwarp();
          }
          double ve = 0.0;
          if (obs) {
            ve = ed;
            for (int k = 1; k <= m_i; ++k) ve = fma(-s_psi[warp][k - 1], sU[32 + lane - k], ve);
          }
          sV[32 + lane] = ve;
          // row set `lane`: t >= m + q and t, t-1, .., t-L observed
          if (lane < hs.n_rs) {
            const uint64_t comb = ((uint64_t)bal << 32) | bprev;
            uint64_t M = comb;
            for (int k = 1; k <= rs_L; ++k) M &= comb << k;
            uint32_t rmask = (uint32_t)(M >> 32);
            if (rs_lo > t0) rmask &= rs_lo - t0 >= 32 ? 0u : ~((1u << (rs_lo - t0)) - 1u);
            n_R += __popc(rmask);
            s_rm[warp][lane] = rmask;
          }
          __syncwarp();
#pragma unroll 1
          for (int e = lane; e < n_ent; e += 32) {
            const uint32_t code = s_code[e];
            uint32_t rm = s_rm[warp][code & 0xffu];
            if (rm == 0u) continue;
            const double* bi = src_base(sE, sV, (code >> 8) & 0xffu);
            const double* bj = src_base(sE, sV, code >> 16);
            double acc = sG[e];
            while (rm) {
              const int j = __ffs(rm) - 1;
              rm &= rm - 1u;
              acc = fma(bi[j], bj[j], acc);
            }
            sG[e] = acc;
          }
          __syncwarp();
          hr_rings_shift(sE, sU, sV, ed);
          bprev = bal;
          __syncwarp();
        }
      }
      __syncthreads();
    }
  }

  // ---- solve: arma_kernel's in-order float64 Cholesky, beta = G^-1 b and the gate, one candidate per lane.  Entry
  // (i, j), i <= j, of the candidate's system is entry (x_i, x_j) of its row set: the e lags, the eps^ lags, the target
  const int nRc = __shfl_sync(0xffffffffu, n_R, rs);
  bool ok = hr_ok && cand && nRc > nreg;
  float f[AR_MAX], th[MA_MAX];
  {
    double w[NR], diag[NR], Lw[NR * NR];
    auto x_of = [&](int i) { return i < p ? i : (i < nreg ? pmax + i - p : pmax + q); };
    auto G = [&](int i, int j) {                                   // i <= j
      const int xi = x_of(i), xj = x_of(j);
      return sG[off + xj * (xj + 1) / 2 + xi];
    };
    for (int j = 0; j < nreg && ok; ++j) {
      double dj = G(j, j);
      for (int k = 0; k < j; ++k) dj -= Lw[j * NR + k] * Lw[j * NR + k];
      if (!(dj > (double)MMF_HR_PIVOT_TOL * G(j, j))) { ok = false; break; }
      diag[j] = sqrt(dj);
      for (int i = j + 1; i < nreg; ++i) {
        double v = G(j, i);
        for (int k = 0; k < j; ++k) v -= Lw[i * NR + k] * Lw[j * NR + k];
        Lw[i * NR + j] = v / diag[j];
      }
    }
    if (ok) {
      for (int i = 0; i < nreg; ++i) {
        double v = G(i, nreg);
        for (int k = 0; k < i; ++k) v -= Lw[i * NR + k] * w[k];
        w[i] = v / diag[i];
      }
      for (int i = nreg - 1; i >= 0; --i) {
        double v = w[i];
        for (int k = i + 1; k < nreg; ++k) v -= Lw[k * NR + i] * w[k];
        w[i] = v / diag[i];
      }
      double fa[AR_MAX], fm[MA_MAX];
      for (int i = 0; i < p; ++i) fa[i] = w[i];
      for (int i = 0; i < q; ++i) fm[i] = -w[p + i];
      ok = step_down_ok(fa, p) && step_down_ok(fm, q);
    }
#pragma unroll
    for (int k = 0; k < AR_MAX; ++k) f[k] = ok && k < p ? (float)w[k] : 0.f;
#pragma unroll
    for (int k = 0; k < MA_MAX; ++k) th[k] = ok && k < q ? (float)w[p + k] : 0.f;
  }
#if MMF_ARMASEL_STOP_AFTER == 2
  if (live && cand && hs.theta != nullptr) hs.theta[row * MA_MAX + lane % MA_MAX] = th[0] + f[0];
  return;                                  // timing build: passes A, A2 and the solve only
#endif

  // ---- scoring walk: each gated candidate lane forecasts the held-out levels [TL, TL + n_hold) dynamically from
  // origin TL with its own recursion from s = 0 (held-out y enters neither the recursion nor the level chain), in pass
  // B's fp32 orders: on a chunk whose 32 rows are all observed fit rows, pass B's lane-parallel AR part and serial MA
  // part; otherwise its all-serial step
  const bool walk = __any_sync(0xffffffffu, ok);
  double sse = 0.0;
  int cnt = 0;
  if (__syncthreads_or(walk)) {
    const int hend = TL + sel.n_hold;      // level rows read: [0, hend)
    const int hendz = hend - dd;
    float hu[AR_MAX], he[MA_MAX];          // hu[k] = u_{s-1-k}, he[k] = eps~_{s-1-k} of this lane's candidate
#pragma unroll
    for (int k = 0; k < AR_MAX; ++k) hu[k] = 0.f;
#pragma unroll
    for (int k = 0; k < MA_MAX; ++k) he[k] = 0.f;
    float l1 = qnan(), l2 = qnan();  // this lane's filled levels ytilde_{t-1}, ytilde_{t-2}
    if (walk && dd > 0) {
      const float v1 = __ldg(yr + dd - 1);
      const float v2 = dd >= 2 ? __ldg(yr + dd - 2) : qnan();
      l1 = finite_f(v1) ? v1 : qnan();
      l2 = finite_f(v2) ? v2 : qnan();
    }
    for (int c0 = 0; c0 < hendz; c0 += TC) {
      stage(s_a, s_nz, d, ar, c0);
      __syncthreads();
      if (walk) {
#pragma unroll 1
        for (int t0 = c0; t0 < min(c0 + TC, hendz); t0 += 32) {
          const int s = t0 + lane;
          const float fit = fitted(s_a, s - c0, g, c);
          const float zv = s < T ? __ldg(zr + s) : 0.f;        // a.y is never read at or beyond its t_fit
          const bool obs = s < T && finite_f(zv);
          const float e = obs ? zv - fit : 0.f;
          const uint32_t bal = __ballot_sync(0xffffffffu, obs);
          const float lv = s + dd < hend ? __ldg(yr + s + dd) : 0.f;   // y is never read at or beyond TL + n_hold
          const bool full = bal == 0xffffffffu;
          const int jn = min(32, hendz - t0);
#pragma unroll 1
          for (int j = 0; j < jn; ++j) {
            const float ej = __shfl_sync(0xffffffffu, e, j);
            const float fj = __shfl_sync(0xffffffffu, fit, j);
            const float yj = __shfl_sync(0xffffffffu, lv, j);
            float arv = 0.f;
#pragma unroll
            for (int k = 0; k < AR_MAX; ++k)
              if (k < p) arv = fmaf(f[k], hu[k], arv);
            float pr, uj, xj;
            if (full) {                                          // pass B's lane-parallel AR part, serial MA part
              const float wj = ej - arv;
              float mj = 0.f;
#pragma unroll
              for (int k = 0; k < MA_MAX; ++k)
                if (k < q) mj = fmaf(th[k], he[k], mj);
              xj = wj - mj;
              pr = arv + mj;
              uj = ej;
            } else {                                             // pass B's all-serial step
              float pj = arv;
#pragma unroll
              for (int k = 0; k < MA_MAX; ++k)
                if (k < q) pj = fmaf(th[k], he[k], pj);
              const bool oj = (bal >> j) & 1u;
              pr = pj;
              uj = oj ? ej : pj;
              xj = oj ? ej - pj : 0.f;
            }
            const float zh = fj + pr;
            const float hj = dd == 0 ? zh : integrate(zh, l1, l2, dd);
            const int tj = t0 + j + dd;                          // level row
            if (tj >= TL && finite_f(yj) && finite_f(hj)) {      // held-out row: score the dynamic forecast
              const double df = (double)yj - (double)hj;
              sse = fma(df, df, sse);
              ++cnt;
            }
#ifdef MMF_ARMASEL_ONE_STEP
            // negative control: an observed held-out value enters the candidate's histories, a leaky one-step score
            if (tj >= TL && finite_f(yj)) {
              if (dd == 0) { uj = yj - fj; xj = uj - pr; }
            }
            const float nl = finite_f(yj) ? yj : hj;
#else
            const float nl = tj < TL && finite_f(yj) ? yj : hj;
#endif
            l2 = l1;
            l1 = nl;
#pragma unroll
            for (int k = AR_MAX - 1; k > 0; --k) hu[k] = hu[k - 1];
            hu[0] = uj;
#pragma unroll
            for (int k = MA_MAX - 1; k > 0; --k) he[k] = he[k - 1];
            he[0] = xj;
          }
        }
      }
      __syncthreads();
    }
  }
  const double mse = ok && cnt > 0 ? sse / (double)cnt : dnan();

  // ---- this launch's first minimum in list order (q, then p), then strictly below the running best.  A candidate that
  // fails the gate forecasts as (p, d, 0), whose score the running best already holds: it never leads
  int win = -1;
  double best = 0.0;
  for (int j = 0; j < hs.n_pq; ++j) {
    const double v = __shfl_sync(0xffffffffu, mse, j);
    if (!isnan(v) && (win < 0 || v < best)) { best = v; win = j; }
  }
  const bool had = (rb.flags & ARIMASEL_SCORED) != 0;
  const bool lead = work && win >= 0 && (!had || best < rb.mse);
  if (win < 0) win = 0;
  const int pw = __shfl_sync(0xffffffffu, p, win), qw = __shfl_sync(0xffffffffu, q, win);
  const int rsw = __shfl_sync(0xffffffffu, rs, win);
  const int nRw = __shfl_sync(0xffffffffu, n_R, rsw);
#pragma unroll
  for (int k = 0; k < AR_MAX; ++k) f[k] = __shfl_sync(0xffffffffu, f[k], win);
#pragma unroll
  for (int k = 0; k < MA_MAX; ++k) th[k] = __shfl_sync(0xffffffffu, th[k], win);

  if (live) {
    // scores: the q = 0 block from arima_select_kernel's scratch; a q >= 1 candidate that fails the gate or is not
    // eligible forecasts as (p, d, 0) and gets its score bit for bit
    if (hs.cand_mse != nullptr) {
      const float* src = hs.cand_q0 + (row * sel.n_diffs + sel.d_index) * sel.n_cand;
      float* dst = hs.cand_mse + (row * sel.n_diffs + sel.d_index) * hs.n_mas * sel.n_cand;
      if (lane < sel.n_cand) dst[lane] = src[lane];
      if (cand) dst[hs.pq_qi[ci] * sel.n_cand + hs.pq_j[ci]] = ok ? (float)mse : src[hs.pq_j[ci]];
    }
    if (lead) {
      if (lane == 0) {
        rb.mse = best; rb.p = (int16_t)pw; rb.d = (int16_t)dd; rb.flags |= ARIMASEL_SCORED;
        sel.best[row] = rb;
        if (sel.choice_p != nullptr) sel.choice_p[row] = pw;
        if (sel.choice_d != nullptr) sel.choice_d[row] = dd;
        if (hs.choice_q != nullptr) hs.choice_q[row] = qw;
        if (sel.mse != nullptr) sel.mse[row] = (float)best;
        if (ar.order != nullptr) ar.order[row] = pw;
        if (hs.ma_order != nullptr) hs.ma_order[row] = qw;
        if (sel.status != nullptr) sel.status[row] = st;
      }
      if (ar.phi != nullptr && lane < AR_MAX) {
        float v = 0.f;
#pragma unroll
        for (int k = 0; k < AR_MAX; ++k) v = lane == k ? f[k] : v;
        ar.phi[row * AR_MAX + lane] = v;
      }
      if (hs.theta != nullptr && lane < MA_MAX) {
        float v = 0.f;
#pragma unroll
        for (int k = 0; k < MA_MAX; ++k) v = lane == k ? th[k] : v;
        hs.theta[row * MA_MAX + lane] = v;
      }
      // the requested levels t < d, which have no prediction
      const int n_nan = min(a.n_pred, dd - a.pred_start);
      for (int k = lane; k < n_nan; k += 32) a.out[row * a.ld_out + k] = qnan();
    } else if (q0_lead || first) {
      // the leader has q = 0 (arima_select_kernel of this d wrote its other outputs), or no candidate is eligible yet
      if (lane == 0) {
        if (hs.choice_q != nullptr) hs.choice_q[row] = q0_lead ? 0 : -1;
        if (hs.ma_order != nullptr) hs.ma_order[row] = 0;
      }
      if (hs.theta != nullptr && lane < MA_MAX) hs.theta[row * MA_MAX + lane] = 0.f;
    }
  }

#if MMF_ARMASEL_STOP_AFTER == 3
  return;                                  // timing build: everything but pass B
#endif
  // ---- pass B with the winner, for the rows this launch leads: arma_kernel's, over the z-space rows [0, max(endz, T))
  if (!__syncthreads_or(lead)) return;
  const int Lb = max(pw, qw);
  const int r_lo = m + qw;
  const int endB = max(endz, T);
  float uprev = 0.f;                       // u of the previous 32 rows
  float he[MA_MAX];                        // he[k] = eps~_{s-1-k}, the same on every lane
#pragma unroll
  for (int k = 0; k < MA_MAX; ++k) he[k] = 0.f;
  double sseB = 0.0;
  bprev = 0u;
  float l1 = qnan(), l2 = qnan();
  if (lead && dd > 0) {
    const float v1 = __ldg(yr + dd - 1);
    const float v2 = dd >= 2 ? __ldg(yr + dd - 2) : qnan();
    l1 = finite_f(v1) ? v1 : qnan();
    l2 = finite_f(v2) ? v2 : qnan();
  }
  for (int c0 = 0; c0 < endB; c0 += TC) {
    stage(s_a, s_nz, d, ar, c0);
    __syncthreads();
    if (lead) {
#pragma unroll 1
      for (int t0 = c0; t0 < min(c0 + TC, endB); t0 += 32) {
        const int s = t0 + lane;
        const float fit = fitted(s_a, s - c0, g, c);
        const float yv = s < T ? __ldg(zr + s) : 0.f;            // never read at or beyond the fit rows
        const bool obs = s < T && finite_f(yv);
        const float e = obs ? yv - fit : 0.f;
        const uint32_t bal = __ballot_sync(0xffffffffu, obs);
        float u, pr, eps = 0.f;
        if (bal == 0xffffffffu) {                                // every row a fit row: AR part lane-parallel
          u = e;
          float arv = 0.f;
#pragma unroll
          for (int k = 1; k <= AR_MAX; ++k)
            if (k <= pw) arv = fmaf(f[k - 1], lagged(u, uprev, k, lane), arv);
          const float w = e - arv;                               // eps~_s = w_s - sum theta_k eps~_{s-k}
          float mav = 0.f;
#pragma unroll 1
          for (int j = 0; j < 32; ++j) {
            float mj = 0.f;
#pragma unroll
            for (int k = 0; k < MA_MAX; ++k)
              if (k < qw) mj = fmaf(th[k], he[k], mj);
            const float ej = __shfl_sync(0xffffffffu, w, j) - mj;
#pragma unroll
            for (int k = MA_MAX - 1; k > 0; --k) he[k] = he[k - 1];
            he[0] = ej;
            if (lane == j) { eps = ej; mav = mj; }
          }
          pr = arv + mav;
        } else {                                                 // a missing or forecast row: all serial
          float hu[AR_MAX];
#pragma unroll
          for (int k = 0; k < AR_MAX; ++k) hu[k] = __shfl_sync(0xffffffffu, uprev, 31 - k);
          u = 0.f; pr = 0.f;
          const int jn = min(32, endB - t0);
#pragma unroll 1
          for (int j = 0; j < jn; ++j) {
            float pj = 0.f;
#pragma unroll
            for (int k = 0; k < AR_MAX; ++k)
              if (k < pw) pj = fmaf(f[k], hu[k], pj);
#pragma unroll
            for (int k = 0; k < MA_MAX; ++k)
              if (k < qw) pj = fmaf(th[k], he[k], pj);
            const float ej = __shfl_sync(0xffffffffu, e, j);
            const bool oj = (bal >> j) & 1u;
            const float uj = oj ? ej : pj;
            const float xj = oj ? ej - pj : 0.f;
#pragma unroll
            for (int k = AR_MAX - 1; k > 0; --k) hu[k] = hu[k - 1];
            hu[0] = uj;
#pragma unroll
            for (int k = MA_MAX - 1; k > 0; --k) he[k] = he[k - 1];
            he[0] = xj;
            if (lane == j) { u = uj; pr = pj; eps = xj; }
          }
        }
        uprev = u;
        if (t0 < T) {                                            // sigma: eps~ over R
          const uint64_t comb = ((uint64_t)bal << 32) | bprev;
          uint64_t M = comb;
          for (int k = 1; k <= Lb; ++k) M &= comb << k;
          const bool inR = ((M >> (32 + lane)) & 1u) && s >= r_lo;
          if (inR) sseB = fma((double)eps, (double)eps, sseB);
          bprev = bal;
        }
        const float zh = fit + pr;
        const int t = s + dd;
        float yh = zh;                                           // d = 0: the level step is the identity
        if (dd > 0) {
          const float lv = t < TL ? __ldg(yr + t) : 0.f;         // y is never read at or beyond t_fit
          const bool lobs = t < TL && finite_f(lv);
          const uint32_t lbal = __ballot_sync(0xffffffffu, lobs);
          if (lbal == 0xffffffffu) {
            const float p1 = __shfl_up_sync(0xffffffffu, lv, 1), p2 = __shfl_up_sync(0xffffffffu, lv, 2);
            yh = integrate(zh, lane >= 1 ? p1 : l1, lane >= 2 ? p2 : (lane == 1 ? l1 : l2), dd);
            l1 = __shfl_sync(0xffffffffu, lv, 31);
            l2 = __shfl_sync(0xffffffffu, lv, 30);
          } else {
            yh = 0.f;
            const int jn = min(32, endB - t0);
#pragma unroll 1
            for (int j = 0; j < jn; ++j) {
              const float hj = integrate(__shfl_sync(0xffffffffu, zh, j), l1, l2, dd);
              const float yj = __shfl_sync(0xffffffffu, lv, j);
              const float nl = (lbal >> j) & 1u ? yj : hj;
              if (lane == j) yh = hj;
              l2 = l1;
              l1 = nl;
            }
          }
        }
        if (t >= a.pred_start && t < end) a.out[row * a.ld_out + (t - a.pred_start)] = yh;
      }
    }
    __syncthreads();
  }
  sseB = warp_sum(sseB);
  if (lead && lane == 0 && ar.sigma != nullptr) ar.sigma[row] = (float)sqrt(sseB / (double)nRw);
}

// Normal-equation entries of the list orders = {p : bit p of order_bits}, mas = {0} and {q : bit q - 1 of ma_bits}, by
// select_arima_call's rule: every (p, q >= 1) pair joins row set R(q, L = max(p, q)), whose p_max is the largest p
// in it, and a row set keeps (p_max + q + 1)(p_max + q + 2) / 2 - 1 entries.
constexpr int armasel_entries(int order_bits, int ma_bits) {
  int pmax[MMF_MA_MAX + 1][MMF_AR_MAX + 1] = {};   // p_max + 1 of R(q, L); 0: no such row set
  for (int q = 1; q <= MMF_MA_MAX; ++q)
    for (int p = 0; p <= MMF_AR_MAX; ++p)
      if ((ma_bits >> (q - 1) & 1) && (order_bits >> p & 1)) {
        int& r = pmax[q][p > q ? p : q];
        r = r > p + 1 ? r : p + 1;
      }
  int n = 0;
  for (int q = 1; q <= MMF_MA_MAX; ++q)
    for (int L = 0; L <= MMF_AR_MAX; ++L)
      if (pmax[q][L] > 0) n += (pmax[q][L] + q) * (pmax[q][L] + q + 1) / 2 - 1;
  return n;
}

constexpr int popcount_c(int v) { return v ? (v & 1) + popcount_c(v >> 1) : 0; }

// the most entries of any list the ABI accepts: orders a nonempty subset of 0..MMF_AR_MAX, mas {0} plus a nonempty
// subset of 1..MMF_MA_MAX, at most MMF_ARMASEL_MAX_PQ pairs (p, q >= 1)
constexpr int armasel_max_entries() {
  int best = 0;
  for (int o = 1; o < 1 << (MMF_AR_MAX + 1); ++o)
    for (int m = 1; m < 1 << MMF_MA_MAX; ++m)
      if (popcount_c(o) * popcount_c(m) <= MMF_ARMASEL_MAX_PQ) {
        const int e = armasel_entries(o, m);
        best = best > e ? best : e;
      }
  return best;
}

constexpr int ARMASEL_MAX_ENT = armasel_max_entries();
// (1..8) x (0..4): 26 row sets; (0..8) x (0..3) (769 entries) and the reference grid (215) stay below 48 KB
static_assert(ARMASEL_MAX_ENT == 1099, "the largest accepted (orders, mas) list has 1,099 entries (74,732 B)");
static_assert(armasel_entries(0x1f, 0xf) == 215 && armasel_entries(0x1ff, 0x7) == 769, "DESIGN.md section 4.18");

}  // namespace

size_t arma_select_smem_bytes(int n_ent) { return (size_t)n_ent * (WARPS * sizeof(double) + sizeof(uint32_t)); }

cudaError_t launch_arma_select(const DesignView& d, const FitArgs& a, const ArArgs& ar, const ArimaArgs& ma,
                               const ArimaSelArgs& sel, const ArmaSelArgs& hs, cudaStream_t s) {
  if (a.n <= 0) return cudaSuccess;
  if (hs.n_ent > ARMASEL_MAX_ENT) return cudaErrorInvalidValue;
  const size_t smem = arma_select_smem_bytes(hs.n_ent);
  if (smem > 48 * 1024) {
    // the attribute is per function and process-wide: always the same value, the largest any call needs, so that a
    // context on another host thread cannot lower it between this call's set and its launch
    const cudaError_t e = cudaFuncSetAttribute(arma_select_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                               (int)arma_select_smem_bytes(ARMASEL_MAX_ENT));
    if (e != cudaSuccess) return e;
  }
  const int64_t grid = (a.n + WARPS - 1) / WARPS;
  arma_select_kernel<<<(unsigned)grid, THREADS, smem, s>>>(d, a, ar, ma, sel, hs);
  return cudaGetLastError();
}

}  // namespace mmf
