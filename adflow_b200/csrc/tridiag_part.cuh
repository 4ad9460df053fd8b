// tridiag_part.cuh -- partitioned Thomas algorithm for ONE tridiagonal system spread over P lanes of a warp
// (Wang's partition method): the lane that owns rows s..e of  a_i x_{i-1} + b_i x_i + c_i x_{i+1} = d_i
//   1. eliminates the sub-diagonal downwards inside its chunk (fill-in: the column of the previous chunk's last
//      unknown y_{p-1}), 2. eliminates the super-diagonal upwards (fill-in: the column of its own last unknown
//   y_p), 3. removes the coupling of its last row to the next chunk's first unknown with that chunk's first row
//   (one warp shuffle), which leaves a tridiagonal system of size P in the y_p, 4. solves that reduced system
//   (every lane redundantly, inputs by shuffles), 5. back-substitutes its interior rows independently.
// The serial chain is about 2 n/P + 2 P divisions instead of 2 n; the arithmetic differs from the reference's
// sequential tridiagsolve (residuals.F90:1750-1783) only by re-association; its error against the exact solution is
// measured in DESIGN.md (after the kernel table) and held by tests/test_line_solves_gpu.py.
//
// Lane mapping inside a warp: lane = p * LS + lineInWarp, LS = 32 / P lines per warp, so that for lines that are
// adjacent in memory (j- and k-direction lines) the LS lanes of equal p read LS consecutive doubles.
#pragma once

template <int P, int M>
struct PartThomas {
    static constexpr int LS = 32 / P;

    // rows of chunk p of a system with n rows: [start, start + len)
    __device__ static __forceinline__ void chunk(int n, int p, int& start, int& len) {
        start = (int)(((long long)p * n) / P);
        len = (int)(((long long)(p + 1) * n) / P) - start;
    }

    // in: a, b, c, d rows 0..m-1 of this lane's chunk (a of the global first row and c of the global last row
    // must be 0); out: the solution overwrites d.  All 32 lanes of the warp must call it (m >= 2 for every chunk).
    __device__ static __forceinline__ void solve(double (&a)[M], double (&b)[M], double (&c)[M], double (&d)[M], int m, int p,
                                                 int lineInWarp) {
        const unsigned full = 0xffffffffu;
        // 1. downward elimination; a[t] becomes the coefficient of y_{p-1}.  The last row of the chunk is tracked in
        // scalars (an `if (t == m - 1)` select over the arrays would be turned into a dynamically indexed load and
        // push the arrays into local memory).
        double la = a[0], lb = b[0], lc = c[0], ld = d[0];
#pragma unroll
        for (int t = 1; t < M; t++) {
            if (t < m) {
                const double f = a[t] / b[t - 1];
                a[t] = -f * a[t - 1];
                b[t] = b[t] - f * c[t - 1];
                d[t] = d[t] - f * d[t - 1];
                la = a[t]; lb = b[t]; lc = c[t]; ld = d[t];
            }
        }
        // 2. upward elimination of rows m-3 .. 0; c[t] becomes the coefficient of y_p (row m-2 already has it)
#pragma unroll
        for (int t = M - 3; t >= 0; t--) {
            if (t <= m - 3) {
                const double f = c[t] / b[t + 1];
                a[t] = a[t] - f * a[t + 1];
                c[t] = -f * c[t + 1];
                d[t] = d[t] - f * d[t + 1];
            }
        }
        // 3. reduced row of this chunk: A y_{p-1} + B y_p + R y_{p+1} = D
        const int next = (p + 1 < P ? p + 1 : p) * LS + lineInWarp;
        const double na = __shfl_sync(full, a[0], next), nb = __shfl_sync(full, b[0], next), nc = __shfl_sync(full, c[0], next),
                     nd = __shfl_sync(full, d[0], next);
        double A = la, B = lb, R = 0.0, D = ld;
        if (p + 1 < P) {
            const double f = lc / nb;
            B = lb - f * na;
            R = -f * nc;
            D = ld - f * nd;
        }
        // 4. reduced system, solved redundantly by every lane
        double rb[P], rr[P], rd[P];
#pragma unroll
        for (int q = 0; q < P; q++) {
            const int src = q * LS + lineInWarp;
            const double qa = __shfl_sync(full, A, src);
            rb[q] = __shfl_sync(full, B, src);
            rr[q] = __shfl_sync(full, R, src);
            rd[q] = __shfl_sync(full, D, src);
            if (q > 0) {
                const double f = qa / rb[q - 1];
                rb[q] = rb[q] - f * rr[q - 1];
                rd[q] = rd[q] - f * rd[q - 1];
            }
        }
        double yn = rd[P - 1] / rb[P - 1];   // y_{P-1}
        double yp = 0.0, ym = 0.0;           // y_p and y_{p-1} of this lane, picked up as scalars on the way
        if (p == P - 1) yp = yn;
        if (p - 1 == P - 1) ym = yn;
#pragma unroll
        for (int q = P - 2; q >= 0; q--) {
            yn = (rd[q] - rr[q] * yn) / rb[q];
            if (q == p) yp = yn;
            if (q == p - 1) ym = yn;
        }
        // 5. interior rows
#pragma unroll
        for (int t = 0; t < M; t++) {
            const double v = (d[t] - a[t] * ym - c[t] * yp) / b[t];
            d[t] = (t < m - 1) ? v : yp;   // rows >= m are padding (b = 1)
        }
    }
};
