// part_thomas_harness.cu -- the partitioned Thomas solver of adflow_b200/csrc/tridiag_part.cuh on its own, for
// tests/test_line_solves_gpu.py.  Built at test time (nvcc, sm_90a) and loaded with ctypes; never linked into the library.
//
// k_part<P, M> solves nLines independent systems  a_t x_{t-1} + b_t x_t + c_t x_{t+1} = d_t  of n rows each, stored line
// after line (row t of line q at q * n + t), with the lane mapping of k_sa_thomas_part (sa_kernels.cuh): lane = p * LS +
// lineInWarp, chunk p of a line from PartThomas::chunk, a of the global first row and c of the global last row set to 0,
// padding rows t >= m of a chunk b = 1 and 0 elsewhere, and lanes past the last line redoing the last line without storing.
#include "../../adflow_b200/csrc/adfb_common.cuh"
#include "../../adflow_b200/csrc/tridiag_part.cuh"

template <int P, int M>
__global__ void __launch_bounds__(32) k_part(const double* __restrict__ ga, const double* __restrict__ gb, const double* __restrict__ gc,
                                             const double* __restrict__ gd, double* __restrict__ gx, int n, int nLines) {
    typedef PartThomas<P, M> PT;
    const int lane = threadIdx.x, p = lane / PT::LS, lw = lane % PT::LS;
    int line = blockIdx.x * PT::LS + lw;
    const bool valid = line < nLines;
    if (!valid) line = nLines - 1;
    const long long base = (long long)line * n;
    int start, m;
    PT::chunk(n, p, start, m);
    double ra[M], rb[M], rc[M], rd[M];
#pragma unroll
    for (int t = 0; t < M; t++) {
        ra[t] = 0.0; rb[t] = 1.0; rc[t] = 0.0; rd[t] = 0.0;
        if (t < m) {
            const long long r = base + start + t;
            ra[t] = (start + t > 0) ? ga[r] : 0.0;
            rb[t] = gb[r];
            rc[t] = (start + t < n - 1) ? gc[r] : 0.0;
            rd[t] = gd[r];
        }
    }
    PT::solve(ra, rb, rc, rd, m, p, lw);
    if (!valid) return;
#pragma unroll
    for (int t = 0; t < M; t++)
        if (t < m) gx[base + start + t] = rd[t];
}

// start and length of every chunk of an n-row system, as the device computes them: out[2 p], out[2 p + 1]
template <int P, int M>
__global__ void k_chunks(int n, int* out) {
    const int p = threadIdx.x;
    if (p >= P) return;
    int start, len;
    PartThomas<P, M>::chunk(n, p, start, len);
    out[2 * p] = start;
    out[2 * p + 1] = len;
}

namespace {
template <int P, int M>
int run(const double* ha, const double* hb, const double* hc, const double* hd, double* hx, int n, int nLines, size_t guard) {
    const size_t sz = (size_t)n * nLines, bytes = sz * sizeof(double);
    double *a = nullptr, *b = nullptr, *c = nullptr, *d = nullptr, *x = nullptr;
    cudaError_t e = cudaSuccess;
    if ((e = cudaMalloc(&a, bytes)) || (e = cudaMalloc(&b, bytes)) || (e = cudaMalloc(&c, bytes)) || (e = cudaMalloc(&d, bytes)) ||
        (e = cudaMalloc(&x, bytes + guard * sizeof(double))))
        goto done;
    if ((e = cudaMemcpy(a, ha, bytes, cudaMemcpyHostToDevice)) || (e = cudaMemcpy(b, hb, bytes, cudaMemcpyHostToDevice)) ||
        (e = cudaMemcpy(c, hc, bytes, cudaMemcpyHostToDevice)) || (e = cudaMemcpy(d, hd, bytes, cudaMemcpyHostToDevice)) ||
        (e = cudaMemcpy(x, hx, bytes + guard * sizeof(double), cudaMemcpyHostToDevice)))   // hx: the poison the caller chose
        goto done;
    k_part<P, M><<<(nLines + PartThomas<P, M>::LS - 1) / PartThomas<P, M>::LS, 32>>>(a, b, c, d, x, n, nLines);
    if ((e = cudaGetLastError()) || (e = cudaDeviceSynchronize())) goto done;
    e = cudaMemcpy(hx, x, bytes + guard * sizeof(double), cudaMemcpyDeviceToHost);
done:
    cudaFree(a); cudaFree(b); cudaFree(c); cudaFree(d); cudaFree(x);
    return (int)e;
}

template <int P, int M>
int chunks(int n, int* hout) {
    int* o = nullptr;
    cudaError_t e = cudaMalloc(&o, 2 * P * sizeof(int));
    if (e) return (int)e;
    k_chunks<P, M><<<1, 32>>>(n, o);
    if (!(e = cudaGetLastError()) && !(e = cudaDeviceSynchronize())) e = cudaMemcpy(hout, o, 2 * P * sizeof(int), cudaMemcpyDeviceToHost);
    cudaFree(o);
    return (int)e;
}
}  // namespace

extern "C" {
// adfb_part_lanes of the library: 8, 16 or 0 (one thread per line) lanes for a line of nl cells
int harness_part_lanes(int nl) { return adfb_part_lanes(nl); }

// x (n * nLines + guard doubles, poisoned by the caller) <- the solution of the nLines systems by PartThomas<P, M>; the guard
// doubles after the last line come back as the caller left them unless a lane stored out of bounds.  -1: no such
// instantiation; otherwise the CUDA error code (0: success).
int harness_part_thomas(int P, int M, const double* a, const double* b, const double* c, const double* d, double* x, int n, int nLines,
                        int guard) {
    if (P == 8 && M == 12) return run<8, 12>(a, b, c, d, x, n, nLines, (size_t)guard);
    if (P == 8 && M == 16) return run<8, 16>(a, b, c, d, x, n, nLines, (size_t)guard);
    if (P == 16 && M == 16) return run<16, 16>(a, b, c, d, x, n, nLines, (size_t)guard);
    return -1;
}

// out[2 p], out[2 p + 1] <- PartThomas<P, M>::chunk(n, p) on the device
int harness_part_chunks(int P, int M, int n, int* out) {
    if (P == 8 && M == 12) return chunks<8, 12>(n, out);
    if (P == 8 && M == 16) return chunks<8, 16>(n, out);
    if (P == 16 && M == 16) return chunks<16, 16>(n, out);
    return -1;
}
}
