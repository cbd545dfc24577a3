// solve_math.cuh -- per-series normal equations of a series with gaps, for ONE thread (registers only).
//
// Shared by solve_rows_kernel (thread-per-series pass over queued records) and by the epilogue warp group of
// fit_tc_kernel (inline, while the next tile streams).  Reference: the fit of build_tune_and_score_model
// (02:435-481) restricted to the observed rows; spec in DESIGN.md section 2:
//   G_i = diag(kept) - sum_{t missing} a_t a_t^T            136 packed entries
//   in-order Cholesky with relative pivot dropping (MMF_PIVOT_TOL), L z = b, L^T gamma = z
#pragma once
#include "mmf_internal.cuh"

namespace mmf {

__device__ __forceinline__ constexpr int tri(int i, int j) { return i * (i + 1) / 2 + j; }   // i >= j

__device__ __forceinline__ void ldg32b_nc(const float* p, float4& lo, float4& hi) {      // p: 32-B aligned (one sector)
  lo = __ldg(reinterpret_cast<const float4*>(p));
  hi = __ldg(reinterpret_cast<const float4*>(p) + 1);
}

// b (moments over the observed rows) -> gamma, in place.  `load_group(seg, gi)` returns the gi-th 8-B group of four
// gap positions of segment seg (SolveRec layout).  Returns the bit mask of columns dropped for rank deficiency.
// `tail(G, outmask, zz)` runs last with the factor L still in G (packed, dropped columns: L_jj = 1, rest 0), the mask
// of unused columns and zz = |z|^2 = b'gamma of the forward solve L z = b (what the standard errors need).
template <class LoadGroup, class Tail>
__device__ __forceinline__ unsigned masked_solve(const DesignView& d, float (&b)[P], int nm0, int nm1,
                                                 LoadGroup load_group, Tail tail) {
  float G[NPAIR];
#pragma unroll
  for (int e = 0; e < NPAIR; ++e) G[e] = 0.f;
#pragma unroll
  for (int j = 0; j < P; ++j) G[tri(j, j)] = ((d.kept_mask >> j) & 1u) ? 1.f : 0.f;
  // software-pipelined: gap positions arrive four at a time (one 8-B load, two groups ahead) and the design row
  // of the next gap is in flight while the 136 FMAs of the current one issue.  Every lane gathers a different
  // 64-B design row (two 32-B sectors).
  auto design_row = [&](int t, float4& r0, float4& r1, float4& r2, float4& r3) {
    const float* ap = d.apred + (size_t)t * P;
    ldg32b_nc(ap, r0, r1);
    ldg32b_nc(ap + 8, r2, r3);
  };
  // (one flat loop over both segments, to pay the warp's max-over-lanes trip count once, measured slower:
  //  the segment-switch bookkeeping costs more issue slots than the shorter trip count saves)
#pragma unroll 1
  for (int seg = 0; seg < 2; ++seg) {
    const int cnt = seg ? nm1 : nm0;
    if (cnt == 0) continue;
    const int n_grp = (cnt + 3) >> 2;
    unsigned long long cur = load_group(seg, 0);
    unsigned long long nxt = n_grp > 1 ? load_group(seg, 1) : 0ull;
    float4 n0, n1, n2, n3;
    design_row((int)(cur & 0xffffull), n0, n1, n2, n3);
#pragma unroll 1
    for (int m = 0; m < cnt; ++m) {
      const float4 a0 = n0, a1 = n1, a2 = n2, a3 = n3;
      const int k1 = (m + 1) & 3;
      if (k1 == 0) {
        cur = nxt;
        const int gi = ((m + 1) >> 2) + 1;
        nxt = gi < n_grp ? load_group(seg, gi) : 0ull;
      }
      // past the end: row 0 is a harmless filler (loaded, never used)
      design_row(m + 1 < cnt ? (int)((cur >> (16 * k1)) & 0xffffull) : 0, n0, n1, n2, n3);
      const float av[P] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w, a2.x, a2.y, a2.z, a2.w, a3.x, a3.y, a3.z, a3.w};
#pragma unroll
      for (int r = 0; r < P; ++r)
#pragma unroll
        for (int q = 0; q <= r; ++q) G[tri(r, q)] = fmaf(-av[r], av[q], G[tri(r, q)]);
    }
  }

  // ---- in-order right-looking Cholesky with pivot dropping (dropped column: L_jj = 1, rest 0)
  unsigned outmask = ~d.kept_mask & 0xFFFFu;
  unsigned dropped = 0u;
  float diag0[P];
#pragma unroll
  for (int j = 0; j < P; ++j) diag0[j] = G[tri(j, j)];
#pragma unroll
  for (int j = 0; j < P; ++j) {
    const float dj = G[tri(j, j)];
    const bool kept_cal = (d.kept_mask >> j) & 1u;
    const bool keep = kept_cal && diag0[j] > 0.f && dj > MMF_PIVOT_TOL * diag0[j];
    if (!keep) {
      outmask |= 1u << j;
      if (kept_cal && diag0[j] > 0.f) dropped |= 1u << j;
    }
    const float inv = keep ? rsqrtf(dj) : 0.f;
    G[tri(j, j)] = keep ? dj * inv : 1.f;
#pragma unroll
    for (int r = j + 1; r < P; ++r) G[tri(r, j)] *= inv;             // column j of L (zero when dropped)
#pragma unroll
    for (int r = j + 1; r < P; ++r)
#pragma unroll
      for (int q = j + 1; q <= r; ++q) G[tri(r, q)] = fmaf(-G[tri(r, j)], G[tri(q, j)], G[tri(r, q)]);
  }
  // ---- L z = b, L^T gamma = z (dropped columns pinned to 0)
#pragma unroll
  for (int j = 0; j < P; ++j) {
    float s = b[j];
#pragma unroll
    for (int q = 0; q < j; ++q) s = fmaf(-G[tri(j, q)], b[q], s);
    b[j] = ((outmask >> j) & 1u) ? 0.f : s / G[tri(j, j)];
  }
  float zz = 0.f;
#pragma unroll
  for (int j = 0; j < P; ++j) zz = fmaf(b[j], b[j], zz);
#pragma unroll
  for (int j = P - 1; j >= 0; --j) {
    float s = b[j];
#pragma unroll
    for (int r = j + 1; r < P; ++r) s = fmaf(-G[tri(r, j)], b[r], s);
    b[j] = ((outmask >> j) & 1u) ? 0.f : s / G[tri(j, j)];
  }
  tail(G, outmask, zz);
  return dropped;
}

// h = |L^-1 a|^2 over the used columns (G as handed to masked_solve's tail; rinv[j] = 1 / L_jj, 0 for an unused column):
// one forward substitution, no division (the reciprocals are taken once per series, not once per prediction row)
__device__ __forceinline__ float leverage_packed(const float (&G)[NPAIR], const float (&rinv)[P], const float (&av)[P]) {
  float w[P];
  float h = 0.f;
#pragma unroll
  for (int j = 0; j < P; ++j) {
    float s = av[j];
#pragma unroll
    for (int q = 0; q < j; ++q) s = fmaf(-G[tri(j, q)], w[q], s);
    w[j] = s * rinv[j];
    h = fmaf(w[j], w[j], h);
  }
  return h;
}

}  // namespace mmf
