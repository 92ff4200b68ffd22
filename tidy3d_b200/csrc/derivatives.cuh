// Derivative pass: first-order perturbation of the eigenvalue lambda = -n^2 of the diagonal operator (oracle/mode_derivatives.py
// is the float64 model).  The left eigenvector is w = G J Q v with J [a; b] = [b; -a] and G the product of the complex-stretched
// primal and dual cell lengths (PMC wall: first dual length halved), so one pass over the Ritz vectors, the coefficient fields
// and the 1-D coefficients gives, per (problem, mode),
//   w^T v,   w^T (f dA/df) v,   sum over cells of (d lambda / d eps_aa) (d eps_aa / df)   (when a dispersion input is given),
// and optionally the per-cell map d n / d eps_{xx,yy,zz}.  A is quadratic in the 1-D coefficients, so f dA/df v is exactly
// [A(c + dc) v - A(c - dc) v] / 2 with dc = f dc/df = -c kappa / s.
#pragma once
#include "kernels.cuh"

namespace b200ms {

constexpr int kDerivChunks = 64;  // blocks per (problem, mode) of the reduction pass

template <typename T, typename C>
struct DerivArgs {
  int nx, ny, num_modes;
  const T *vec;            // sorted Ritz vectors, mode q of problem b at vec + q*vstride + b*2N
  size_t vstride;
  const C *fields;         // exx, eyy, iez, (mxx, myy, imz)
  size_t field_bstride;
  const T *cx, *cy;        // [B][4][n] 1-D coefficients
  const T *dcx, *dcy;      // [B][4][n] f dc/df
  const cplx *gx, *gy;     // [B][2][n] primal / dual stretched lengths (metric of the left eigenvector)
  const double *jz_e;      // [B][jz_len] bend: eps' = diag(1/je, 1/je, je) eps, or null
  int jz_axis, jz_len;
  const cplx *deps;        // [B][3][N] d eps_aa / df of the caller's permittivity (1/Hz), or null
  cplx *partial;           // [B*M][kDerivChunks][3]
  const cplx *scale;       // [B][M] d n / d lambda / (w^T v): map = numerator * scale
  cplx *map;               // [B][3][N][M]
};

template <typename T, typename C, bool HAS_MU>
struct DerivCell {
  DiagSite<T, C, HAS_MU> S;
  const cplx *gx, *gy;
  const double *je;  // this problem's bend factors or null
  int jz_axis;

  // w = G J Q v at (ii, jj); zero outside the grid
  __device__ __forceinline__ void w(int ii, int jj, cplx &w1, cplx &w2) const {
    if (!S.in(ii, jj)) {
      w1 = w2 = mk(0.0, 0.0);
      return;
    }
    T q1, q2, t00;
    S.q(ii, jj, q1, q2, t00);
    const int nx = S.nx, ny = S.ny;
    w1 = (gx[ii] * gy[ny + jj]) * to_cplx(q2);
    w2 = -((gx[nx + ii] * gy[jj]) * to_cplx(q1));
  }
  // z = Dxf^T w1 + Dyf^T w2 at (ii, jj), given w there
  __device__ __forceinline__ cplx z(int ii, int jj, cplx w1, cplx w2) const {
    if (!S.in(ii, jj)) return mk(0.0, 0.0);
    cplx a1, a2, b1, b2;
    w(ii - 1, jj, a1, a2);
    w(ii, jj - 1, b1, b2);
    return to_cplx(S.CX(0, ii)) * w1 + to_cplx(S.CX(1, ii - 1)) * a1 + to_cplx(S.CY(0, jj)) * w2 + to_cplx(S.CY(1, jj - 1)) * b2;
  }
  __device__ __forceinline__ cplx iez(int ii, int jj) const { return S.in(ii, jj) ? to_cplx(ldg(S.iez + (size_t)ii * S.ny + jj)) : mk(0.0, 0.0); }
  // w^T (d A / d eps_aa(i, j)) v of the caller's permittivity (PEC-valued cells: 0)
  __device__ __forceinline__ void eps_grad(int i, int j, cplx w1, cplx w2, cplx d[3]) const {
    const size_t g = (size_t)i * S.ny + j;
    const cplx zg = z(i, j, w1, w2);
    cplx a1, a2, b1, b2;
    w(i + 1, j, a1, a2);
    w(i, j + 1, b1, b2);
    const cplx zx = z(i + 1, j, a1, a2), zy = z(i, j + 1, b1, b2);
    const cplx iz = iez(i, j);
    const cplx mx = HAS_MU ? to_cplx(ldg(S.mxx + g)) : mk(1.0, 0.0), my = HAS_MU ? to_cplx(ldg(S.myy + g)) : mk(1.0, 0.0);
    d[0] = -(to_cplx(S.V1(i, j)) * (to_cplx(S.CX(2, i)) * iz * zg + to_cplx(S.CX(3, i + 1)) * iez(i + 1, j) * zx + my * w1));
    d[1] = -(to_cplx(S.V2(i, j)) * (to_cplx(S.CY(2, j)) * iz * zg + to_cplx(S.CY(3, j + 1)) * iez(i, j + 1) * zy + mx * w2));
    d[2] = -(zg * iz * to_cplx(S.u(i, j)));
    const double pec = 0.9 * 1e8;  // PEC-valued input: stored as 1 + 1e8 i (solver.py:327-333)
    if (abs2(to_cplx(ldg(S.exx + g))) >= pec * pec) d[0] = mk(0.0, 0.0);
    if (abs2(to_cplx(ldg(S.eyy + g))) >= pec * pec) d[1] = mk(0.0, 0.0);
    if (abs2(iz) * pec * pec <= 1.0) d[2] = mk(0.0, 0.0);
    if (je) {  // eps'_xx = eps_xx / je, eps'_yy = eps_yy / je, eps'_zz = je eps_zz
      const double f = je[jz_axis == 0 ? i : j];
      d[0] = d[0] * (1.0 / f);
      d[1] = d[1] * (1.0 / f);
      d[2] = d[2] * f;
    }
  }
};

template <typename T, typename C, bool HAS_MU>
__device__ __forceinline__ DerivCell<T, C, HAS_MU> deriv_cell(const DerivArgs<T, C> &a, int b, int m, const T *dc_x, const T *dc_y, double s) {
  const int nx = a.nx, ny = a.ny;
  const size_t N = (size_t)nx * ny;
  const T *v1 = a.vec + (size_t)m * a.vstride + (size_t)b * 2 * N;
  const C *fb = a.fields + a.field_bstride * b;
  return DerivCell<T, C, HAS_MU>{
      DiagSite<T, C, HAS_MU>{v1, v1 + N, fb, fb + N, fb + 2 * N, fb + 3 * N, fb + 4 * N, fb + 5 * N,
                             CoefRows<T>{a.cx + (size_t)b * 4 * nx, dc_x ? dc_x + (size_t)b * 4 * nx : nullptr, s, nx},
                             CoefRows<T>{a.cy + (size_t)b * 4 * ny, dc_y ? dc_y + (size_t)b * 4 * ny : nullptr, s, ny}, nx, ny},
      a.gx + (size_t)b * 2 * nx, a.gy + (size_t)b * 2 * ny, a.jz_e ? a.jz_e + (size_t)b * a.jz_len : nullptr, a.jz_axis};
}

// grid (kDerivChunks, B*M), 256 threads: partial sums of w^T v, w^T (f dA/df) v and the material term per chunk of cells
template <typename T, typename C, bool HAS_MU>
__global__ void __launch_bounds__(256) deriv_scan_kernel(DerivArgs<T, C> a) {
  const int M = a.num_modes, bm = blockIdx.y, b = bm / M, m = bm % M;
  const int nx = a.nx, ny = a.ny;
  const size_t N = (size_t)nx * ny;
  const DerivCell<T, C, HAS_MU> c0 = deriv_cell<T, C, HAS_MU>(a, b, m, (const T *)nullptr, (const T *)nullptr, 0.0);
  const DerivCell<T, C, HAS_MU> cp = deriv_cell<T, C, HAS_MU>(a, b, m, a.dcx, a.dcy, 1.0), cm = deriv_cell<T, C, HAS_MU>(a, b, m, a.dcx, a.dcy, -1.0);
  const cplx *de = a.deps ? a.deps + (size_t)b * 3 * N : nullptr;
  cplx s_wv = mk(0.0, 0.0), s_da = mk(0.0, 0.0), s_mat = mk(0.0, 0.0);
  for (size_t g = (size_t)blockIdx.x * 256 + threadIdx.x; g < N; g += (size_t)gridDim.x * 256) {
    const int i = (int)(g / ny), j = (int)(g % ny);
    cplx w1, w2;
    c0.w(i, j, w1, w2);
    s_wv += w1 * to_cplx(c0.S.V1(i, j)) + w2 * to_cplx(c0.S.V2(i, j));
    T p1p, p2p, p1m, p2m;
    cp.S.apply(i, j, p1p, p2p);
    cm.S.apply(i, j, p1m, p2m);
    s_da += 0.5 * (w1 * to_cplx(p1p - p1m) + w2 * to_cplx(p2p - p2m));
    if (de) {
      cplx d[3];
      c0.eps_grad(i, j, w1, w2, d);
      s_mat += d[0] * ldg(de + g) + d[1] * ldg(de + N + g) + d[2] * ldg(de + 2 * N + g);
    }
  }
  __shared__ cplx red[3][256];
  red[0][threadIdx.x] = s_wv;
  red[1][threadIdx.x] = s_da;
  red[2][threadIdx.x] = s_mat;
  __syncthreads();
  for (int h = 128; h > 0; h >>= 1) {
    if ((int)threadIdx.x < h)
      for (int k = 0; k < 3; ++k) red[k][threadIdx.x] += red[k][threadIdx.x + h];
    __syncthreads();
  }
  if (threadIdx.x < 3) a.partial[((size_t)bm * gridDim.x + blockIdx.x) * 3 + threadIdx.x] = red[threadIdx.x][0];
}

// one thread per (problem, mode) and sum: the chunks in a fixed order
__global__ void deriv_final_kernel(const cplx *partial, int nchunk, int count, cplx *out) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= count) return;
  const int bm = t / 3, k = t % 3;
  cplx s = mk(0.0, 0.0);
  for (int c = 0; c < nchunk; ++c) s += partial[((size_t)bm * nchunk + c) * 3 + k];
  out[t] = s;
}

// grid like epilogue_kernel: map[b][a][g][m] = (w^T dA/d eps_aa(g) v) * scale[b][m]
template <typename T, typename C, bool HAS_MU>
__global__ void __launch_bounds__(256) deriv_map_kernel(DerivArgs<T, C> a) {
  const int nx = a.nx, ny = a.ny, M = a.num_modes;
  const size_t N = (size_t)nx * ny;
  const int j = blockIdx.x * 64 + threadIdx.x, i = blockIdx.y * 4 + threadIdx.y;
  const int m = blockIdx.z % M, b = blockIdx.z / M;
  if (i >= nx || j >= ny) return;
  const DerivCell<T, C, HAS_MU> c0 = deriv_cell<T, C, HAS_MU>(a, b, m, (const T *)nullptr, (const T *)nullptr, 0.0);
  cplx w1, w2, d[3];
  c0.w(i, j, w1, w2);
  c0.eps_grad(i, j, w1, w2, d);
  const cplx sc = a.scale[(size_t)b * M + m];
  const size_t g = (size_t)i * ny + j;
  cplx *o = a.map + (size_t)b * 3 * N * M;
  for (int k = 0; k < 3; ++k) o[((size_t)k * N + g) * M + m] = d[k] * sc;
}

}  // namespace b200ms
