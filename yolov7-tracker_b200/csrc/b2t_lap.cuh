// b2t_lap.cuh -- exact thresholded linear assignment, one CTA per problem.
//
// Replaces ``lap.lapjv(cost, extend_cost=True, cost_limit=t)`` as called from
// tracker/matching.py:30-41.  lap solves the (N+M)^2 cost-limit-extended square problem
// (oracle/lapjv.py), whose optimum equals
//        minimise  sum_matched (c_ij - t)   over partial matchings,
// so only entries c_ij < t can ever be matched.  With IoU costs that graph is ~99 % empty and
// falls apart into many small connected components (SURVEY.md 7.2 #2), hence:
//   1. the caller hands over the sub-threshold entries as CSR rows (col, cost);
//   2. exact kernelisation in parallel rounds (lap_kernelize): with weights w = t - c > 0 the problem
//      is a maximum-weight matching, and a mutually-best edge (i, j) whose weight exceeds the sum
//      of the second-best weights at i and at j belongs to every optimal matching (exchange
//      argument: any matching without it loses at most those two weights by swapping it in).
//      Such edges are fixed, their endpoints removed, and the rule re-applied until nothing
//      changes -- in tracking this settles the obvious track/detection pairs (most rows) and
//      shatters the big weakly-connected components;
//   3. every remaining row is augmented once by a Jonker-Volgenant-style shortest-augmenting-path search
//      with dual potentials (u, v): one warp per search, lanes over the row's edges for the
//      relaxation and over the frontier for the arg-min;
//   4. the rows that survive are grouped by connected component of the residual graph
//      (min-label propagation, one thread per row, with pointer jumping); component c is solved by
//      warp c mod #warps, its rows in ascending order -- no two warps ever share a column, so
//      there is nothing to lock and the result is deterministic.  A search that outgrows its
//      warp's frontier buffer is retried at the end on one warp with the full-size buffer.
// Rectangular formulation: each row owns a private "stay unmatched" column of cost t/2 (its
// dual never moves, so it is never stored) and real edges are shifted by -t/2 -- every row is
// assigned exactly once (to a real column or to its own dummy), N augmentations in total.
// The result is the unique optimum whenever that is unique (ties are solver-dependent in lap
// as well; the generators are tie-free).
#pragma once
#include <string.h>
#include "b2t_prims.cuh"

namespace b2t {

template <class T> struct LapCsr {
    const int* row_start;   // nullptr -> row i starts at i * row_stride
    int row_stride;
    const int* row_cnt;
    const int* e_col;       // global storage
    const T* e_cost;
    const int* s_col;       // optional shared-memory storage: row i lives there iff start(i) + cnt(i) <= s_cap
    const T* s_cost;
    int s_cap;
    const int* e_row;       // optional: row index of every entry (global / shared), enables the edge-parallel passes
    const int* s_row;
    int n_entries;          // entries [0, n_entries) are exactly the rows' ranges (contiguous CSR), 0 if unknown
    // optional SECOND shared-memory window: the entries [w2_base, w2_end) of the global storage mirrored at index e - w2_base
    // (the fused tracker step copies the first spilled rows into shared memory that is idle during the solve: a Dijkstra step
    // that reads its row from L2 costs ~600 cycles, and a dense association spends thousands of steps there)
    const int* w2_col = nullptr;
    const T* w2_cost = nullptr;
    const int* w2_row = nullptr;
    int w2_base = 0, w2_end = 0;
    B2T_DEV int start(int i) const { return row_start ? row_start[i] : i * row_stride; }
    B2T_DEV bool in_smem(int st, int cnt) const { return st + cnt <= s_cap; }
    B2T_DEV bool in_w2(int st, int cnt) const { return st >= w2_base && st + cnt <= w2_end; }
    B2T_DEV const int* cols(int st, int cnt) const {
        if (in_smem(st, cnt)) return s_col + st;
        if (in_w2(st, cnt)) return w2_col + (st - w2_base);
        return e_col + st;
    }
    B2T_DEV const T* costs(int st, int cnt) const {
        if (in_smem(st, cnt)) return s_cost + st;
        if (in_w2(st, cnt)) return w2_cost + (st - w2_base);
        return e_cost + st;
    }
    // entry e of a contiguous CSR -> (row, col, cost pointer); false when e is not a stored entry
    B2T_DEV bool entry(int e, int n, int& i, int& j, T& c) const {
        i = e < s_cap ? s_row[e] : -1;
        bool sm_ok = false;
        if (i >= 0 && i < n) { const int st = row_start[i], en = st + row_cnt[i]; sm_ok = st <= e && e < en && en <= s_cap; }
        if (sm_ok) { j = s_col[e]; c = s_cost[e]; return true; }
        const bool in2 = e >= w2_base && e < w2_end;          // entries are mirrored one by one: a row may straddle the window's end
        i = in2 ? w2_row[e - w2_base] : e_row[e];
        if (i < 0 || i >= n) return false;
        const int st = row_start[i], en = st + row_cnt[i];
        if (!(st <= e && e < en && en > s_cap)) return false;
        if (in2) { j = w2_col[e - w2_base]; c = w2_cost[e - w2_base]; }
        else { j = e_col[e]; c = e_cost[e]; }
        return true;
    }
};

template <class T> struct LapWork {
    T *u, *v, *dist;
    int *x, *y, *pred, *tl, *q0, *q1, *q2, *cur, *tlw;
    unsigned char *sc, *rdead, *cdead;
    int* scratch;   // 64 ints
    enum { TLC = 64, MAXW = 32 };   // frontier capacity of a warp's search buffer, max warps per CTA
    template <class A> B2T_HD void carve(A& a, int nmax, int mmax) {
        u = a.template take<T>(nmax); v = a.template take<T>(mmax); dist = a.template take<T>(mmax);
        x = a.template take<int>(nmax); y = a.template take<int>(mmax); pred = a.template take<int>(mmax);
        tl = a.template take<int>(mmax);
        q0 = a.template take<int>(nmax); q1 = a.template take<int>(nmax); q2 = a.template take<int>(nmax);
        cur = a.template take<int>(nmax > 2 * 64 ? nmax : 2 * 64); tlw = a.template take<int>(TLC * MAXW);
        sc = a.template take<unsigned char>(mmax); rdead = a.template take<unsigned char>(nmax);
        cdead = a.template take<unsigned char>(mmax); scratch = a.template take<int>(64);
    }
};

#define B2T_LAP_BIG ((T)1e30)
#if defined(B2T_HOSTSIM)
#define B2T_LSUB(idx) do { } while (0)
#else
#define B2T_LSUB(idx) do { if (dbg && threadIdx.x == 0) { const long long n_ = clock64(); dbg[idx] = (int)(n_ - *dbgt); *dbgt = n_; } } while (0)
#endif

// One warp: shortest augmenting path from row r0.  tl / tl_cap: this warp's frontier buffer.
// Returns false -- with every touched entry restored and nothing committed -- when the frontier
// buffer is full.
template <class T>
B2T_DEV bool lap_augment_row(const LapCsr<T>& g, const T half_t, LapWork<T>& w, const int r0, int* tl, const int tl_cap) {
    const int lane = lane_id();
    const unsigned lt = lanemask_lt();
    int nt = 0;
    T minval = (T)0;
    int i = r0;
    T best_dummy = half_t - w.u[r0];
    int dummy_row = r0;
    int sink = -1;   // -1: dummy of dummy_row, >= 0: free real column
    bool failed = false;
    for (;;) {
        const T ui = w.u[i];
        const int es = g.start(i), ec = g.row_cnt[i];
        const int* ecol = g.cols(es, ec);
        const T* ecost = g.costs(es, ec);
        // Two 32-entry chunks per trip, and every chunk's column AND cost are requested before anything is tested: a row that lives
        // in the global workspace then costs ONE L2 round trip per 64 entries instead of a dependent pair per 32.
        for (int e0 = 0; e0 < ec; e0 += 64) {
            int jq[2]; T cq[2]; bool aq[2];
#pragma unroll
            for (int q = 0; q < 2; ++q) {
                const int e = e0 + 32 * q + lane;
                aq[q] = e < ec;
                jq[q] = aq[q] ? ecol[e] : -1;
                cq[q] = aq[q] ? ecost[e] : (T)0;
            }
#pragma unroll
            for (int q = 0; q < 2; ++q) {
                if (e0 + 32 * q >= ec) break;                 // (uniform)
                bool act = aq[q], fresh = false, full = false;
                const int j = jq[q];
                if (act) { if (j < 0 || w.cdead[j] || w.sc[j]) act = false; }
                T red = (T)0;
                if (act) {
                    red = minval + (((cq[q] - half_t) - ui) - w.v[j]);
                    fresh = w.dist[j] >= B2T_LAP_BIG;
                }
                const unsigned fm = __ballot_sync(B2T_FULL, fresh);
                if (fresh) {
                    const int pos = nt + __popc(fm & lt);
                    if (pos < tl_cap) tl[pos] = j; else { full = true; act = false; }
                    // column j joins the frontier: if it is popped, the search continues from the row matched to it.  When that
                    // row's entries live in the global workspace, ask for them now (L1 prefetch)
                    const int yj = w.y[j];
                    if (yj >= 0) {
                        const int s2 = g.start(yj), c2 = g.row_cnt[yj];
                        if (!g.in_smem(s2, c2) && !g.in_w2(s2, c2)) {
                            B2T_PREFETCH_L1(g.e_col + s2);
                            B2T_PREFETCH_L1(g.e_cost + s2);
                            if (c2 > 16) B2T_PREFETCH_L1(g.e_cost + s2 + 16);
                            if (c2 > 32) { B2T_PREFETCH_L1(g.e_col + s2 + 32); B2T_PREFETCH_L1(g.e_cost + s2 + 32); }
                        }
                    }
                }
                if (act && red < w.dist[j]) { w.dist[j] = red; w.pred[j] = i; }
                nt += __popc(fm);
                if (nt > tl_cap) nt = tl_cap;
                if (__any_sync(B2T_FULL, full)) failed = true;
            }
        }
        __syncwarp();
        if (failed) break;
        T cand = B2T_LAP_BIG;
        int cj = -1;
        // (four frontier entries per lane and trip: the loads of a trip are independent, so a long frontier costs one chain of
        // shared-memory latencies per 128 entries instead of one per 32 -- the dense-scene searches spend most of their time here)
        for (int k = lane; k < nt; k += 128) {
            int jj[4]; bool on[4]; T dd[4];
#pragma unroll
            for (int q = 0; q < 4; ++q) { on[q] = k + 32 * q < nt; jj[q] = on[q] ? tl[k + 32 * q] : 0; }
#pragma unroll
            for (int q = 0; q < 4; ++q) { on[q] = on[q] && !w.sc[jj[q]]; dd[q] = w.dist[jj[q]]; }
#pragma unroll
            for (int q = 0; q < 4; ++q)
                if (on[q] && (cj < 0 || dd[q] < cand || (dd[q] == cand && jj[q] < cj))) { cand = dd[q]; cj = jj[q]; }
        }
        T bv = B2T_LAP_BIG;
        const int bj = warp_argmin(cand, cj, &bv);
        if (bj < 0 || best_dummy <= bv) { sink = -1; minval = best_dummy; break; }
        minval = bv;
        if (lane == 0) w.sc[bj] = 1;
        __syncwarp();
        const int yi = w.y[bj];
        if (yi < 0) { sink = bj; break; }
        i = yi;
        const T dd = minval + (half_t - w.u[i]);
        if (dd < best_dummy) { best_dummy = dd; dummy_row = i; }
    }
    if (!failed) {
        // dual update (pre-augmentation y), then flip the path
        for (int k = lane; k < nt; k += 32) {
            const int j = tl[k];
            if (w.sc[j]) {
                const T d = minval - w.dist[j];
                w.v[j] = w.v[j] - d;
                const int yi = w.y[j];
                if (yi >= 0) w.u[yi] = w.u[yi] + d;
            }
        }
        if (lane == 0) w.u[r0] = w.u[r0] + minval;
        __syncwarp();
        if (lane == 0) {
            if (sink < 0) {
                int ii = dummy_row;
                int jprev = w.x[ii];
                w.x[ii] = -1;
                while (ii != r0) {
                    const int j = jprev;
                    ii = w.pred[j];
                    w.y[j] = ii;
                    jprev = w.x[ii];
                    w.x[ii] = j;
                }
            } else {
                int j = sink;
                for (;;) {
                    const int ii = w.pred[j];
                    w.y[j] = ii;
                    const int jn = w.x[ii];
                    w.x[ii] = j;
                    j = jn;
                    if (ii == r0) break;
                }
            }
        }
        __syncwarp();
    }
    for (int k = lane; k < nt; k += 32) { const int j = tl[k]; w.dist[j] = B2T_LAP_BIG; w.sc[j] = 0; }
    __syncwarp();
    return !failed;
}

// Kernelisation keys: the weight rounded to float32, as an order-preserving unsigned (weights are
// positive).  Shared-memory atomicMax is native for 32 bits (the 64-bit form is a CAS loop).
B2T_DEV unsigned int wkey32(float v) { unsigned int k; memcpy(&k, &v, 4); return k; }
B2T_DEV float wval32(unsigned int k) { float v; memcpy(&v, &k, 4); return v; }
// The key of a live edge (weight t - c > 0): at least 1, so that key 0 always means "no edge" -- a
// float64 weight below half of float32's smallest denormal would otherwise round to key 0 and its row
// would be dropped as edgeless.  The clamp is monotone, so the order of the keys is kept.
template <class T> B2T_DEV unsigned int wkey_live(T w) { const unsigned int k = wkey32((float)w); return k ? k : 1u; }
// An upper bound of every weight whose key is k: the next float up.  Rounding to nearest can put
// the key up to half a float ulp BELOW the weight (at weights >= 32 that is more than 2e-6), but
// the next float lies strictly above it.  Key 0 (no edge) gives the smallest denormal; the key of
// +inf (a weight beyond float range) gives NaN, and a comparison with NaN never fixes an edge.
B2T_DEV double wup32(unsigned int k) { return (double)wval32(k + 1u); }

// Exact kernelisation, row-parallel form (any CSR).  An edge (i, j) whose weight W exceeds S_i + S_j,
// where S_i / S_j bound the weight of every OTHER live edge at row i / column j, belongs to every
// optimal matching: a matching without it loses at most S_i + S_j by dropping the edges at i and j
// and gains W by taking (i, j).  The rule fixes a mutually-best edge when
//      (double)t - (double)c_ij  >  wup32(second key at i) + wup32(second key at j)
// in float64, in both instantiations.  Each wup32 lies strictly above its true second best, so
// U = wup32 + wup32 > S_i + S_j exactly.  Each side of the test is ONE rounding of an exact value
// (W = t - c of two floats or two doubles, U of two floats), and rounding is monotone: W <= U
// implies fl(W) <= fl(U).  So a fired test implies W > U > S_i + S_j for any finite weight, with no
// absolute margin.  (The argument holds in float32 arithmetic too; evaluating in float64 makes both
// instantiations take the same decision on a problem whose costs are float32.)  Column-side best / second-best are reduced with 32-bit shared-memory atomics on
// the keys (ties for a column's best go to the smallest row, and the other rows of the tie then set
// the second key to the best key, so the rule cannot fire).  All threads; leaves w.rdead / w.cdead / x / y.
template <class T>
B2T_DEVNI void lap_kernelize_rows(int n, int m, const LapCsr<T>& g, T thresh, LapWork<T>& w) {
    const int tid = (int)threadIdx.x, nthr = (int)blockDim.x;
    unsigned* cb = reinterpret_cast<unsigned*>(w.dist);
    unsigned* cs = reinterpret_cast<unsigned*>(w.v);
    int* cbrow = w.pred;
    for (int round = 0; round < 12; ++round) {
        for (int j = tid; j < m; j += nthr) { cb[j] = 0; cs[j] = 0; cbrow[j] = 0x7fffffff; }
        if (tid == 0) w.scratch[44] = 0;
        __syncthreads();
        for (int i = tid; i < n; i += nthr) {
            if (w.rdead[i]) continue;
            const int es = g.start(i), ec = g.row_cnt[i];
            const int* ecol = g.cols(es, ec);
            const T* ecost = g.costs(es, ec);
            for (int e = 0; e < ec; ++e) { const int j = ecol[e]; if (j >= 0 && !w.cdead[j]) atomicMax(&cb[j], wkey_live<T>(thresh - ecost[e])); }
        }
        __syncthreads();
        for (int i = tid; i < n; i += nthr) {
            if (w.rdead[i]) continue;
            const int es = g.start(i), ec = g.row_cnt[i];
            const int* ecol = g.cols(es, ec);
            const T* ecost = g.costs(es, ec);
            for (int e = 0; e < ec; ++e) { const int j = ecol[e]; if (j >= 0 && !w.cdead[j] && wkey_live<T>(thresh - ecost[e]) == cb[j]) atomicMin(&cbrow[j], i); }
        }
        __syncthreads();
        for (int i = tid; i < n; i += nthr) {
            if (w.rdead[i]) continue;
            const int es = g.start(i), ec = g.row_cnt[i];
            const int* ecol = g.cols(es, ec);
            const T* ecost = g.costs(es, ec);
            for (int e = 0; e < ec; ++e) { const int j = ecol[e]; if (j >= 0 && !w.cdead[j] && cbrow[j] != i) atomicMax(&cs[j], wkey_live<T>(thresh - ecost[e])); }
        }
        __syncthreads();
        for (int i = tid; i < n; i += nthr) {
            if (w.rdead[i]) continue;
            const int es = g.start(i), ec = g.row_cnt[i];
            const int* ecol = g.cols(es, ec);
            const T* ecost = g.costs(es, ec);
            T w1 = (T)0, w2 = (T)0, c1 = (T)0;
            int j1 = -1;
            for (int e = 0; e < ec; ++e) {
                const int j = ecol[e];
                if (j < 0 || w.cdead[j]) continue;
                const T ww = thresh - ecost[e];
                if (ww > w1) { w2 = w1; w1 = ww; j1 = j; c1 = ecost[e]; } else if (ww > w2) w2 = ww;
            }
            if (j1 < 0) { w.rdead[i] = 1; continue; }                          // no live edge left: stays unmatched
            // (the row's second best through its key as well: in float32, t - c may have rounded below its true weight)
            if (cbrow[j1] == i && (double)thresh - (double)c1 > wup32(wkey32((float)w2)) + wup32(cs[j1])) {
                w.x[i] = j1; w.y[j1] = i; w.scratch[44] = 1; w.sc[j1] = 2;
            }
        }
        __syncthreads();
        // retire the fixed pairs in a separate pass: a row testing the rule must not see a column another row fixed in the same
        // pass, or how far a chain of fixes runs in one round would depend on thread timing
        for (int j = tid; j < m; j += nthr) if (w.sc[j] == 2) { w.sc[j] = 0; w.cdead[j] = 1; w.rdead[w.y[j]] = 1; }
        const int changed = w.scratch[44];
        if (tid == 0) w.scratch[46] = round + 1;
        __syncthreads();
        if (!changed) break;
    }
}

// Same rule, EDGE-parallel (contiguous CSR with row indices): one thread per stored entry, best /
// second-best of rows and columns by 32-bit atomics -- no per-row loops, so a high-degree row does
// not stall its warp.  4 short passes per round.
template <class T>
B2T_DEVNI void lap_kernelize_edges(int n, int m, const LapCsr<T>& g, T thresh, LapWork<T>& w) {
    const int tid = (int)threadIdx.x, nthr = (int)blockDim.x;
    const int nE = g.n_entries;
    unsigned* cb = reinterpret_cast<unsigned*>(w.dist);
    unsigned* cs = reinterpret_cast<unsigned*>(w.v);
    unsigned* rb = reinterpret_cast<unsigned*>(w.u);
    unsigned* rs = reinterpret_cast<unsigned*>(w.q1);
    int* cbrow = w.pred;
    int* rbcol = w.q2;
    for (int round = 0; round < 12; ++round) {
        for (int j = tid; j < m; j += nthr) { cb[j] = 0; cs[j] = 0; cbrow[j] = 0x7fffffff; }
        for (int i = tid; i < n; i += nthr) { rb[i] = 0; rs[i] = 0; rbcol[i] = 0x7fffffff; }
        if (tid == 0) w.scratch[44] = 0;
        __syncthreads();
        for (int e = tid; e < nE; e += nthr) {
            int i, j; T c;
            if (!g.entry(e, n, i, j, c) || j < 0 || w.rdead[i] || w.cdead[j]) continue;
            const unsigned k = wkey_live<T>(thresh - c);
            atomicMax(&cb[j], k); atomicMax(&rb[i], k);
        }
        __syncthreads();
        for (int e = tid; e < nE; e += nthr) {
            int i, j; T c;
            if (!g.entry(e, n, i, j, c) || j < 0 || w.rdead[i] || w.cdead[j]) continue;
            const unsigned k = wkey_live<T>(thresh - c);
            if (k == cb[j]) atomicMin(&cbrow[j], i);
            if (k == rb[i]) atomicMin(&rbcol[i], j);
        }
        __syncthreads();
        for (int e = tid; e < nE; e += nthr) {
            int i, j; T c;
            if (!g.entry(e, n, i, j, c) || j < 0 || w.rdead[i] || w.cdead[j]) continue;
            const unsigned k = wkey_live<T>(thresh - c);
            if (cbrow[j] != i) atomicMax(&cs[j], k);
            if (rbcol[i] != j) atomicMax(&rs[i], k);
        }
        for (int i = tid; i < n; i += nthr) if (!w.rdead[i] && rb[i] == 0) w.rdead[i] = 1;   // no live edge left
        __syncthreads();
        for (int e = tid; e < nE; e += nthr) {
            int i, j; T c;
            if (!g.entry(e, n, i, j, c) || j < 0 || w.rdead[i] || w.cdead[j]) continue;
            // the rule of lap_kernelize_rows, with both second bests from keys
            if (cbrow[j] == i && rbcol[i] == j && (double)thresh - (double)c > wup32(rs[i]) + wup32(cs[j])) {
                w.x[i] = j; w.y[j] = i; w.scratch[44] = 1; w.sc[j] = 2;
            }
        }
        __syncthreads();
        // retire the fixed pairs (separate pass: the test pass above must see a consistent dead set)
        for (int j = tid; j < m; j += nthr) if (w.sc[j] == 2) { w.sc[j] = 0; w.cdead[j] = 1; w.rdead[w.y[j]] = 1; }
        const int changed = w.scratch[44];
        if (tid == 0) w.scratch[46] = round + 1;
        __syncthreads();
        if (!changed) break;
    }
    // the arrays borrowed from the solver are re-initialised by the caller (u, q1, q2)
    for (int i = tid; i < n; i += nthr) w.u[i] = (T)0;
    __syncthreads();
}

// All threads of the CTA.  On return w.x[0..n) / w.y[0..m) hold the assignment (-1 = unmatched).
template <class T>
B2T_DEVNI void lap_solve_cta(int n, int m, const LapCsr<T>& g, T thresh, LapWork<T>& w, int* dbg = nullptr, long long* dbgt = nullptr) {
    const int tid = (int)threadIdx.x, nthr = (int)blockDim.x;
    const int lane = lane_id(), wid = warp_id(), nw = num_warps();
    const T half_t = thresh / (T)2;
    for (int i = tid; i < n; i += nthr) { w.u[i] = (T)0; w.x[i] = -1; w.rdead[i] = g.row_cnt[i] > 0 ? 0 : 1; }
    for (int j = tid; j < m; j += nthr) { w.y[j] = -1; w.sc[j] = 0; w.cdead[j] = 0; }
    if (tid < 8) w.scratch[40 + tid] = 0;
    __syncthreads();
    if (n == 0 || m == 0) return;
    B2T_LSUB(0);
    if (g.e_row && g.n_entries > 0) lap_kernelize_edges<T>(n, m, g, thresh, w);
    else lap_kernelize_rows<T>(n, m, g, thresh, w);
    B2T_LSUB(1);
    int* lab_r = w.q2;      // labels of residual rows (row indices)
    int* lab_c = w.tl;      // labels of residual columns
    for (int j = tid; j < m; j += nthr) { w.v[j] = (T)0; w.dist[j] = B2T_LAP_BIG; lab_c[j] = 0x3fffffff; }
    for (int i = tid; i < n; i += nthr) lab_r[i] = i;
    const int nq0 = block_compact(n, [&](int i) { return w.rdead[i] == 0; }, w.q0, w.scratch);
    if (tid == 0) w.scratch[45] = nq0;
    B2T_LSUB(2);
    if (nq0 == 0) return;
    // ---- connected components of the residual graph (min-label propagation with pointer jumping)
    const bool flat = g.e_row && g.n_entries > 0;
    for (;;) {
        if (tid == 0) w.scratch[44] = 0;
        __syncthreads();
        if (flat) {
            for (int e = tid; e < g.n_entries; e += nthr) {
                int i, j; T c;
                if (!g.entry(e, n, i, j, c) || j < 0 || w.rdead[i] || w.cdead[j]) continue;
                int l = lab_r[i];
                const int lc = lab_c[j];
                if (lc < l) l = lc;
                const int lj = lab_r[l];
                if (lj < l) l = lj;
                bool ch = false;
                if (l < lab_r[i]) { atomicMin(&lab_r[i], l); ch = true; }
                if (l < lab_c[j]) { atomicMin(&lab_c[j], l); ch = true; }
                if (ch) w.scratch[44] = 1;
            }
        } else {
            for (int k = tid; k < nq0; k += nthr) {
                const int i = w.q0[k];
                const int es = g.start(i), ec = g.row_cnt[i];
                const int* ecol = g.cols(es, ec);
                const int l0 = lab_r[i];
                int l = l0;
                for (int e = 0; e < ec; ++e) { const int j = ecol[e]; if (j >= 0 && !w.cdead[j]) { const int lc = lab_c[j]; if (lc < l) l = lc; } }
                const int lj = lab_r[l];
                if (lj < l) l = lj;
                bool ch = l < l0;
                if (ch) lab_r[i] = l;
                for (int e = 0; e < ec; ++e) {
                    const int j = ecol[e];
                    if (j >= 0 && !w.cdead[j] && lab_c[j] > l) { atomicMin(&lab_c[j], l); ch = true; }
                }
                if (ch) w.scratch[44] = 1;
            }
        }
        __syncthreads();
        const int changed = w.scratch[44];
        __syncthreads();
        if (!changed) break;
    }
    B2T_LSUB(3);
    // ---- warp (label mod #warps) solves the component, rows ascending; overflowing searches -> q1
    {
        int* tl = w.tlw + wid * LapWork<T>::TLC;
        for (int k = 0; k < nq0; ++k) {
            const int i = w.q0[k];
            if (lab_r[i] % nw != wid) continue;
            if (!lap_augment_row<T>(g, half_t, w, i, tl, LapWork<T>::TLC)) {
                if (lane == 0) w.q1[atomicAdd(&w.scratch[41], 1)] = i;
            }
        }
    }
    __syncthreads();
    B2T_LSUB(4);
    const int nq1 = w.scratch[41];
    if (nq1 > 0) {
        // rare: a search touched more than TLC columns.  One warp, full-size frontier (lab_c is dead now).
        if (wid == 0) {
            // deterministic order
            for (int a = 0; a < nq1; ++a) {
                int best = 0x7fffffff;
                for (int b = lane; b < nq1; b += 32) { const int r = w.q1[b]; if (r >= 0 && r < best) best = r; }
                for (int o = 16; o; o >>= 1) { const int ob = shfl_xor(best, o); if (ob < best) best = ob; }
                for (int b = lane; b < nq1; b += 32) if (w.q1[b] == best) w.q1[b] = -1;
                __syncwarp();
                lap_augment_row<T>(g, half_t, w, best, w.tl, m);
            }
        }
        __syncthreads();
    }
}

}  // namespace b2t
