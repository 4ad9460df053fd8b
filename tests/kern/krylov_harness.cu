// krylov_harness.cu -- the vector kernels of the device GMRES (adflow_b200/csrc/krylov_kernels.cuh) on their own, for
// tests/test_krylov_kernels_gpu.py.  Built at test time (nvcc, sm_90a) and loaded with ctypes; never linked into the library.
//
// Every entry takes host arrays, runs the kernels with the launch configuration adfb_gmres_solve gives them (kry_dots:
// k_multidot over ADFB_GMRES_PARTS CTAs of 256 threads, then k_multidot_final with one CTA per vector; k_axpy_many and
// k_scale_to one thread per entry in CTAs of 256) and returns the CUDA error code (0: success).  The `guard` doubles
// after the n outputs come back as the caller left them unless a thread stored out of bounds.
#include "../../adflow_b200/csrc/adfb_common.cuh"
#include "../../adflow_b200/csrc/krylov_kernels.cuh"

namespace {
struct Dev {
    double* p = nullptr;
    ~Dev() { cudaFree(p); }
};
cudaError_t up(Dev& d, const double* h, size_t count) {
    cudaError_t e = cudaMalloc(&d.p, count * sizeof(double));
    return e ? e : cudaMemcpy(d.p, h, count * sizeof(double), cudaMemcpyHostToDevice);
}
}  // namespace

extern "C" {
// out[i] = V_i . w for i < nv, V_i at V + i * ld (nv * ld doubles), as kry_dots forms the Gram-Schmidt projections
int harness_dots(const double* V, long long ld, int nv, const double* w, long long n, double* out) {
    if (nv < 1 || nv > ADFB_GMRES_MAXV || ld < n) return -1;
    Dev dV, dw, dred;
    cudaError_t e;
    if ((e = up(dV, V, (size_t)nv * ld)) || (e = up(dw, w, (size_t)n)) ||
        (e = cudaMalloc(&dred.p, ((size_t)ADFB_GMRES_PARTS + 1) * ADFB_GMRES_MAXV * sizeof(double))))
        return (int)e;
    double* fin = dred.p + (size_t)ADFB_GMRES_PARTS * ADFB_GMRES_MAXV;
    k_multidot<<<ADFB_GMRES_PARTS, 256>>>(dV.p, ld, nv, dw.p, n, dred.p);
    k_multidot_final<<<nv, 256>>>(dred.p, ADFB_GMRES_PARTS, nv, fin);
    if ((e = cudaGetLastError()) || (e = cudaDeviceSynchronize())) return (int)e;
    return (int)cudaMemcpy(out, fin, nv * sizeof(double), cudaMemcpyDeviceToHost);
}

// y[q] <- beta y[q] + sum_i coef[i] V_i[q] for q < n; y holds n + guard doubles
int harness_axpy_many(const double* V, long long ld, int nv, const double* coef, double beta, double* y, long long n, int guard) {
    if (nv < 0 || nv > ADFB_GMRES_MAXV || ld < n) return -1;
    GmresCoef c = {};
    for (int i = 0; i < nv; i++) c.c[i] = coef[i];
    Dev dV, dy;
    cudaError_t e;
    if ((e = up(dV, V, (size_t)(nv > 0 ? nv : 1) * ld)) || (e = up(dy, y, (size_t)n + guard))) return (int)e;
    k_axpy_many<<<(unsigned)((n + 255) / 256), 256>>>(dV.p, ld, nv, c, beta, dy.p, n);
    if ((e = cudaGetLastError()) || (e = cudaDeviceSynchronize())) return (int)e;
    return (int)cudaMemcpy(y, dy.p, ((size_t)n + guard) * sizeof(double), cudaMemcpyDeviceToHost);
}

// y[q] <- a x[q] for q < n; y holds n + guard doubles
int harness_scale_to(const double* x, double a, double* y, long long n, int guard) {
    Dev dx, dy;
    cudaError_t e;
    if ((e = up(dx, x, (size_t)n)) || (e = up(dy, y, (size_t)n + guard))) return (int)e;
    k_scale_to<<<(unsigned)((n + 255) / 256), 256>>>(dx.p, a, dy.p, n);
    if ((e = cudaGetLastError()) || (e = cudaDeviceSynchronize())) return (int)e;
    return (int)cudaMemcpy(y, dy.p, ((size_t)n + guard) * sizeof(double), cudaMemcpyDeviceToHost);
}
}
