// Derivative pass: first-order perturbation of the eigenvalue lambda = -n^2 of the diagonal operator (oracle/mode_derivatives.py
// is the float64 model).  The left eigenvector is w = G J Q v with J [a; b] = [b; -a] and G the product of the complex-stretched
// primal and dual cell lengths (PMC wall: first dual length halved), so one pass over the Ritz vectors, the coefficient fields
// and the 1-D coefficients gives, per (problem, mode),
//   w^T v,   w^T (f dA/df) v,   sum over cells of (d lambda / d eps_aa) (d eps_aa / df)   (when a dispersion input is given),
// and optionally the per-cell map d n / d eps_{xx,yy,zz}.  A is quadratic in the 1-D coefficients, so f dA/df v is exactly
// [A(c + dc) v - A(c - dc) v] / 2 with dc = f dc/df = -c kappa / s.
#pragma once
#include "kernels.cuh"
#include "medium.cuh"

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

// ------------------------------------------------------------------------------------------------
// Perturbation responses (b200ms_pert): the permittivity gradients contracted against caller-given fields delta eps_k without
// writing the maps.  The perturbations of a device batch sit at eps + k kstride + b bstride ([ncomp][N] each; bstride 0 when
// every problem passes the same field).  The first-order scans sum (per-site gradient) . delta eps_k over a grid-stride chunk
// for kPertGroup perturbations at a time; the per-site kernels of the group and dispersion passes evaluate their forms once per
// site and reduce each form . delta eps_k over the block (pert_site_sums).  Every sum of one perturbation is formed in the
// same order whichever other perturbations share its launch or its device group, and deriv_final_kernel adds the chunks or
// blocks in a fixed order.
// ------------------------------------------------------------------------------------------------
struct PertArgs {
  const cplx *eps;        // delta eps of perturbation k of problem b at eps + k kstride + b bstride, [ncomp][N]
  size_t kstride, bstride;
  int npert;              // perturbations of this launch
  cplx *partial;          // scans: [B*M][kPertGroup / 3][nchunk][3]; per-site kernels: [B][rows][nblock][3]
};
constexpr int kPertGroup = 6;  // perturbations per launch of the first-order scans (accumulators per thread)

// grid (kDerivChunks, B*M), 256 threads: per chunk, sum_g sum_a (w^T dA/d eps_aa(g) v) delta eps_k,a(g) for k < p.npert
template <typename T, typename C, bool HAS_MU>
__global__ void __launch_bounds__(256) deriv_pert_kernel(DerivArgs<T, C> a, PertArgs p) {
  const int M = a.num_modes, bm = blockIdx.y, b = bm / M, m = bm % M;
  const int ny = a.ny;
  const size_t N = (size_t)a.nx * ny;
  const DerivCell<T, C, HAS_MU> c0 = deriv_cell<T, C, HAS_MU>(a, b, m, (const T *)nullptr, (const T *)nullptr, 0.0);
  const cplx *pe = p.eps + p.bstride * b;
  cplx s[kPertGroup];
#pragma unroll
  for (int k = 0; k < kPertGroup; ++k) s[k] = mk(0.0, 0.0);
  for (size_t g = (size_t)blockIdx.x * 256 + threadIdx.x; g < N; g += (size_t)gridDim.x * 256) {
    const int i = (int)(g / ny), j = (int)(g % ny);
    cplx w1, w2, d[3];
    c0.w(i, j, w1, w2);
    c0.eps_grad(i, j, w1, w2, d);
#pragma unroll
    for (int k = 0; k < kPertGroup; ++k)
      if (k < p.npert) {
        const cplx *e = pe + k * p.kstride + g;
        s[k] += d[0] * ldg(e) + d[1] * ldg(e + N) + d[2] * ldg(e + 2 * N);
      }
  }
  __shared__ cplx red[kPertGroup][256];
  for (int k = 0; k < kPertGroup; ++k) red[k][threadIdx.x] = s[k];
  __syncthreads();
  for (int h = 128; h > 0; h >>= 1) {
    if ((int)threadIdx.x < h)
      for (int k = 0; k < kPertGroup; ++k) red[k][threadIdx.x] += red[k][threadIdx.x + h];
    __syncthreads();
  }
  if (threadIdx.x < kPertGroup)
    p.partial[(((size_t)bm * (kPertGroup / 3) + threadIdx.x / 3) * gridDim.x + blockIdx.x) * 3 + threadIdx.x % 3] = red[threadIdx.x][0];
}

// Block sums of the NF per-site forms f[v][a] (a: xx, yy, zz) of site g of problem b against every perturbation of p:
// value v + NF k of problem b, sum over the block of sum_a f[v][a] delta eps_k,a(g), goes to
// p.partial[((b rows + (v + NF k) / 3) nblock + block) 3 + (v + NF k) % 3] with rows = ceil(NF npert / 3) (the padding: 0).
// Every thread of the block calls it; `live` is false for threads outside the grid.
template <int NF>
__device__ __forceinline__ void pert_site_sums(const PertArgs &p, int b, size_t g, size_t N, bool live, const cplx (&f)[NF][3]) {
  __shared__ cplx red[256];
  const int t = threadIdx.y * blockDim.x + threadIdx.x, nblk = gridDim.x * gridDim.y, blk = blockIdx.y * gridDim.x + blockIdx.x;
  const int rows = (NF * p.npert + 2) / 3;
  const cplx *e = p.eps + p.bstride * b + g;
#pragma unroll 1
  for (int k = 0; k < p.npert; ++k) {
#pragma unroll
    for (int v = 0; v < NF; ++v) {
      cplx s = mk(0.0, 0.0);
      if (live) {
        const cplx *ek = e + k * p.kstride;
        s = f[v][0] * ldg(ek) + f[v][1] * ldg(ek + N) + f[v][2] * ldg(ek + 2 * N);
      }
      red[t] = s;
      __syncthreads();
      for (int h = 128; h > 0; h >>= 1) {
        if (t < h) red[t] += red[t + h];
        __syncthreads();
      }
      const int o = NF * k + v;
      if (t == 0) p.partial[(((size_t)b * rows + o / 3) * nblk + blk) * 3 + o % 3] = red[0];
      __syncthreads();
    }
  }
  for (int o = NF * p.npert + t; o < 3 * rows; o += 256) p.partial[(((size_t)b * rows + o / 3) * nblk + blk) * 3 + o % 3] = mk(0.0, 0.0);
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

// ------------------------------------------------------------------------------------------------
// Dispersion pass: the second frequency derivative of lambda (oracle/mode_dispersion.py is the float64 model).  In the scaled
// direction ' = f d/df, with p = (exx, eyy, 1/ezz) of the solver frame and c the 1-D coefficients (A has degree <= 2 in each),
//   A'v  = [A(c+c',p) - A(c-c',p)]/2 + [A(c,p+p') - A(c,p-p')]/2,
//   A''v = A(c+c',p) + A(c-c',p) + A(c,p+p') + A(c,p-p') - 4 A(c,p) + [A(c+c'',p) - A(c-c'',p)]/2 + [A(c,p+p'') - A(c,p-p'')]/2
//          + [A(c+c',p+p') - A(c+c',p-p') - A(c-c',p+p') + A(c-c',p-p')]/2
// are exact with unit steps.  Per mode slot, phase 0 sums w^T v, w^T A'v and w^T A''v; phase 1 writes the projected right-hand
// side r = -(A'v - beta v), beta = w^T A'v / w^T v, of the correction solve (A - lambda) x = r; phase 2 sums w^T x and
// w^T A'x.  Then lambda'' = [w^T A''v + 2 (w^T A'x - lambda' w^T x)] / w^T v (the v-component of x drops out).
// ------------------------------------------------------------------------------------------------

// (A(c + sc dc, p + sp dp) v)(i, j) in double-complex arithmetic (the perturbations may be complex for a real operator)
template <typename T, typename C, bool HAS_MU>
struct PertSite {
  const T *v1, *v2;
  const C *fb;       // this problem's coefficient fields: exx, eyy, iez, mxx, myy, imz at fb + k N
  const cplx *dp;    // this problem's [3][N] direction of (exx, eyy, iez), or null
  double sp;
  CoefRows<T> CX, CY;
  int nx, ny;
  size_t N;
  __device__ __forceinline__ bool in(int ii, int jj) const { return ii >= 0 && ii < nx && jj >= 0 && jj < ny; }
  __device__ __forceinline__ cplx V1(int ii, int jj) const { return in(ii, jj) ? to_cplx(ldg(v1 + (size_t)ii * ny + jj)) : mk(0.0, 0.0); }
  __device__ __forceinline__ cplx V2(int ii, int jj) const { return in(ii, jj) ? to_cplx(ldg(v2 + (size_t)ii * ny + jj)) : mk(0.0, 0.0); }
  __device__ __forceinline__ cplx cx(int w, int i) const { return to_cplx(CX(w, i)); }
  __device__ __forceinline__ cplx cy(int w, int j) const { return to_cplx(CY(w, j)); }
  __device__ __forceinline__ cplx fld(int k, size_t g) const {
    cplx e = to_cplx(ldg(fb + (size_t)k * N + g));
    if (dp) e += sp * ldg(dp + (size_t)k * N + g);
    return e;
  }
  __device__ __forceinline__ cplx TT(int ii, int jj) const {
    if (!in(ii, jj)) return mk(0.0, 0.0);
    cplx acc = cx(0, ii) * V2(ii, jj) + cx(1, ii) * V2(ii + 1, jj) - cy(0, jj) * V1(ii, jj) - cy(1, jj) * V1(ii, jj + 1);
    if (HAS_MU) acc = to_cplx(ldg(fb + 5 * N + (size_t)ii * ny + jj)) * acc;
    return acc;
  }
  __device__ __forceinline__ cplx u(int i, int j) const {
    if (!in(i, j)) return mk(0.0, 0.0);
    const size_t g = (size_t)i * ny + j;
    cplx uacc = cx(2, i) * (fld(0, g) * V1(i, j)) + cy(2, j) * (fld(1, g) * V2(i, j));
    if (i > 0) uacc += cx(3, i) * (fld(0, g - ny) * V1(i - 1, j));
    if (j > 0) uacc += cy(3, j) * (fld(1, g - 1) * V2(i, j - 1));
    return -(fld(2, g) * uacc);
  }
  __device__ __forceinline__ void apply(int i, int j, cplx &p1, cplx &p2) const {
    const size_t g = (size_t)i * ny + j;
    const cplx t00 = TT(i, j);
    const cplx q1 = cx(2, i) * t00 + cx(3, i) * TT(i - 1, j) + fld(1, g) * V2(i, j);
    const cplx q2 = cy(2, j) * t00 + cy(3, j) * TT(i, j - 1) - fld(0, g) * V1(i, j);
    const cplx u0 = u(i, j);
    p1 = cx(0, i) * u0 + cx(1, i) * u(i + 1, j);
    p2 = cy(0, j) * u0 + cy(1, j) * u(i, j + 1);
    if (HAS_MU) {
      p1 += to_cplx(ldg(fb + 4 * N + g)) * q2;
      p2 -= to_cplx(ldg(fb + 3 * N + g)) * q1;
    } else {
      p1 += q2;
      p2 -= q1;
    }
  }
};

// one operator evaluation of the difference formulas above: coefficient direction (0 none, 1 c', 2 c'') and step, field
// direction (0 none, 1 p', 2 p'') and step, weight in A'v and in A''v
struct DispTerm {
  int cdir, pdir;
  double sc, sp, w1, w2;
};
__constant__ DispTerm kDispTermsP[13] = {  // dispersive media
    {1, 0, 1.0, 0.0, 0.5, 1.0},  {1, 0, -1.0, 0.0, -0.5, 1.0}, {0, 1, 0.0, 1.0, 0.5, 1.0},  {0, 1, 0.0, -1.0, -0.5, 1.0},
    {0, 0, 0.0, 0.0, 0.0, -4.0}, {2, 0, 1.0, 0.0, 0.0, 0.5},   {2, 0, -1.0, 0.0, 0.0, -0.5}, {0, 2, 0.0, 1.0, 0.0, 0.5},
    {0, 2, 0.0, -1.0, 0.0, -0.5}, {1, 1, 1.0, 1.0, 0.0, 0.5},  {1, 1, 1.0, -1.0, 0.0, -0.5}, {1, 1, -1.0, 1.0, 0.0, -0.5},
    {1, 1, -1.0, -1.0, 0.0, 0.5}};
__constant__ DispTerm kDispTermsC[5] = {  // nondispersive media: only the coefficients move
    {1, 0, 1.0, 0.0, 0.5, 1.0}, {1, 0, -1.0, 0.0, -0.5, 1.0}, {0, 0, 0.0, 0.0, 0.0, -2.0}, {2, 0, 1.0, 0.0, 0.0, 0.5}, {2, 0, -1.0, 0.0, 0.0, -0.5}};

template <typename T, typename C>
struct DispArgs {
  DerivArgs<T, C> d;    // Ritz vectors, coefficient fields, 1-D coefficients, f dc/df, metric and bend factors of the first-order pass
  const T *c2x, *c2y;   // [B][4][n] f^2 d^2c/df^2 = 2 (f dc/df)^2 / c
  const cplx *p1, *p2;  // [B][3][N] f dp/df and f^2 d^2p/df^2, or both null (nondispersive batch)
  int q;                // mode slot
  const T *x;           // phase 2: the correction, batched-vector layout
  T *r;                 // phase 1: the right-hand side, batched-vector layout
  const cplx *beta;     // phase 1: [B] w^T A'v / w^T v
  cplx *partial;        // [B][nchunk][3]
};

// grid (nchunk, B), 256 threads; phases as described above
template <typename T, typename C, bool HAS_MU>
__global__ void __launch_bounds__(256) disp_scan_kernel(DispArgs<T, C> a, int phase) {
  const int b = blockIdx.y, nx = a.d.nx, ny = a.d.ny;
  const size_t N = (size_t)nx * ny;
  const bool hp = a.p1 != nullptr;
  const DispTerm *tab = hp ? kDispTermsP : kDispTermsC;
  const int nterm = phase == 0 ? (hp ? 13 : 5) : (hp ? 4 : 2);
  const T *vec = phase == 2 ? a.x + (size_t)b * 2 * N : a.d.vec + (size_t)a.q * a.d.vstride + (size_t)b * 2 * N;
  const T *cxb = a.d.cx + (size_t)b * 4 * nx, *cyb = a.d.cy + (size_t)b * 4 * ny;
  const T *d1x = a.d.dcx + (size_t)b * 4 * nx, *d1y = a.d.dcy + (size_t)b * 4 * ny;
  const T *d2x = a.c2x + (size_t)b * 4 * nx, *d2y = a.c2y + (size_t)b * 4 * ny;
  const cplx *p1 = hp ? a.p1 + (size_t)b * 3 * N : nullptr, *p2 = hp ? a.p2 + (size_t)b * 3 * N : nullptr;
  const C *fb = a.d.fields + a.d.field_bstride * b;
  const cplx beta = phase == 1 ? a.beta[b] : mk(0.0, 0.0);
  cplx s0 = mk(0.0, 0.0), s1 = mk(0.0, 0.0), s2 = mk(0.0, 0.0);
  for (size_t g = (size_t)blockIdx.x * 256 + threadIdx.x; g < N; g += (size_t)gridDim.x * 256) {
    const int i = (int)(g / ny), j = (int)(g % ny);
    cplx w1 = mk(0.0, 0.0), w2 = mk(0.0, 0.0);
    if (phase != 1) deriv_cell<T, C, HAS_MU>(a.d, b, a.q, (const T *)nullptr, (const T *)nullptr, 0.0).w(i, j, w1, w2);
    cplx a1x = mk(0.0, 0.0), a1y = mk(0.0, 0.0), a2x = mk(0.0, 0.0), a2y = mk(0.0, 0.0);
#pragma unroll 1
    for (int t = 0; t < nterm; ++t) {
      const DispTerm tm = tab[t];
      const T *dcx = tm.cdir == 1 ? d1x : (tm.cdir == 2 ? d2x : nullptr), *dcy = tm.cdir == 1 ? d1y : (tm.cdir == 2 ? d2y : nullptr);
      const PertSite<T, C, HAS_MU> P{vec, vec + N, fb, tm.pdir == 1 ? p1 : (tm.pdir == 2 ? p2 : nullptr), tm.sp,
                                     CoefRows<T>{cxb, dcx, tm.sc, nx}, CoefRows<T>{cyb, dcy, tm.sc, ny}, nx, ny, N};
      cplx y1, y2;
      P.apply(i, j, y1, y2);
      a1x += tm.w1 * y1;
      a1y += tm.w1 * y2;
      a2x += tm.w2 * y1;
      a2y += tm.w2 * y2;
    }
    const cplx e1 = to_cplx(ldg(vec + g)), e2 = to_cplx(ldg(vec + N + g));
    if (phase == 1) {
      T *rb = a.r + (size_t)b * 2 * N;
      rb[g] = cast_to<T>(-(a1x - beta * e1));
      rb[N + g] = cast_to<T>(-(a1y - beta * e2));
      continue;
    }
    s0 += w1 * e1 + w2 * e2;
    s1 += w1 * a1x + w2 * a1y;
    s2 += w1 * a2x + w2 * a2y;
  }
  if (phase == 1) return;
  __shared__ cplx red[3][256];
  red[0][threadIdx.x] = s0;
  red[1][threadIdx.x] = s1;
  red[2][threadIdx.x] = s2;
  __syncthreads();
  for (int h = 128; h > 0; h >>= 1) {
    if ((int)threadIdx.x < h)
      for (int k = 0; k < 3; ++k) red[k][threadIdx.x] += red[k][threadIdx.x + h];
    __syncthreads();
  }
  if (threadIdx.x < 3) a.partial[((size_t)b * gridDim.x + blockIdx.x) * 3 + threadIdx.x] = red[threadIdx.x][0];
}

// [B][3][N] f dp/df and f^2 d^2p/df^2 of p = (exx, eyy, iez) in the solver frame from d eps / df and d^2 eps / df^2 of the caller's
// diagonal (in place: dp1 holds d eps / df on entry, dp2 d^2 eps / df^2).  Bend: exx = eps_xx / je, eyy = eps_yy / je,
// ezz = je eps_zz; freq: [B] Hz.  iez' = -ezz' iez^2, iez'' = 2 ezz'^2 iez^3 - ezz'' iez^2.  PEC-valued cells: 0 (as eps_grad).
// With dp3 (the third-order pass): dp3 holds d^3 eps / df^3 on entry and receives f^3 d^3p/df^3, iez''' = -ezz''' iez^2 +
// 6 ezz' ezz'' iez^3 - 6 ezz'^3 iez^4, and dps / dpd receive the combined directions p' + p'' and p' - p''.  With dp4 as well (the
// fourth-order pass): dp4 holds d^4 eps / df^4 on entry and receives f^4 d^4p/df^4, iez'''' = -ezz'''' iez^2 + (8 ezz' ezz''' +
// 6 ezz''^2) iez^3 - 36 ezz'^2 ezz'' iez^4 + 24 ezz'^4 iez^5, and dqs / dqd receive p' + p''' and p' - p'''.
template <typename C>
__global__ void disp_fields_kernel(int nx, int ny, int B, const C *fields, size_t field_bstride, const double *jz_e, int jz_axis, int jz_len,
                                   const double *freq, cplx *dp1, cplx *dp2, cplx *dp3, cplx *dps, cplx *dpd, cplx *dp4, cplx *dqs,
                                   cplx *dqd) {
  const size_t N = (size_t)nx * ny;
  for (size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x; t < (size_t)B * N; t += (size_t)gridDim.x * blockDim.x) {
    const int b = (int)(t / N);
    const size_t g = t % N;
    const int i = (int)(g / ny), j = (int)(g % ny);
    const double f = freq[b];
    const C *fb = fields + field_bstride * b;
    const double je = jz_e ? jz_e[(size_t)b * jz_len + (jz_axis == 0 ? i : j)] : 1.0;
    cplx *d1 = dp1 + (size_t)b * 3 * N + g, *d2 = dp2 + (size_t)b * 3 * N + g;
    const double pec = 0.9 * 1e8;
    const cplx iz = to_cplx(ldg(fb + 2 * N + g));
    for (int k = 0; k < 2; ++k) {
      const bool is_pec = abs2(to_cplx(ldg(fb + (size_t)k * N + g))) >= pec * pec;
      d1[(size_t)k * N] = is_pec ? mk(0.0, 0.0) : d1[(size_t)k * N] * (f / je);
      d2[(size_t)k * N] = is_pec ? mk(0.0, 0.0) : d2[(size_t)k * N] * (f * f / je);
    }
    const cplx e1 = d1[2 * N] * (f * je), e2 = d2[2 * N] * (f * f * je);  // f ezz', f^2 ezz''
    const bool is_pec = abs2(iz) * pec * pec <= 1.0;
    const cplx iz2 = iz * iz;
    d1[2 * N] = is_pec ? mk(0.0, 0.0) : -(e1 * iz2);
    d2[2 * N] = is_pec ? mk(0.0, 0.0) : 2.0 * (e1 * e1) * (iz2 * iz) - e2 * iz2;
    if (!dp3) continue;
    cplx *d3 = dp3 + (size_t)b * 3 * N + g, *ds = dps + (size_t)b * 3 * N + g, *dd = dpd + (size_t)b * 3 * N + g;
    for (int k = 0; k < 2; ++k) {
      const bool pk = abs2(to_cplx(ldg(fb + (size_t)k * N + g))) >= pec * pec;
      d3[(size_t)k * N] = pk ? mk(0.0, 0.0) : d3[(size_t)k * N] * (f * f * f / je);
    }
    const cplx e3 = d3[2 * N] * (f * f * f * je);  // f^3 ezz'''
    d3[2 * N] = is_pec ? mk(0.0, 0.0) : 6.0 * (e1 * e2) * (iz2 * iz) - e3 * iz2 - 6.0 * (e1 * e1 * e1) * (iz2 * iz2);
    for (int k = 0; k < 3; ++k) {
      ds[(size_t)k * N] = d1[(size_t)k * N] + d2[(size_t)k * N];
      dd[(size_t)k * N] = d1[(size_t)k * N] - d2[(size_t)k * N];
    }
    if (!dp4) continue;
    cplx *d4 = dp4 + (size_t)b * 3 * N + g, *qs = dqs + (size_t)b * 3 * N + g, *qd = dqd + (size_t)b * 3 * N + g;
    const double f4 = (f * f) * (f * f);
    for (int k = 0; k < 2; ++k) {
      const bool pk = abs2(to_cplx(ldg(fb + (size_t)k * N + g))) >= pec * pec;
      d4[(size_t)k * N] = pk ? mk(0.0, 0.0) : d4[(size_t)k * N] * (f4 / je);
    }
    const cplx e4 = d4[2 * N] * (f4 * je);  // f^4 ezz''''
    const cplx iz3 = iz2 * iz, iz4 = iz2 * iz2;
    d4[2 * N] = is_pec ? mk(0.0, 0.0)
                       : (8.0 * (e1 * e3) + 6.0 * (e2 * e2)) * iz3 - e4 * iz2 - 36.0 * (e1 * e1 * e2) * iz4 + 24.0 * ((e1 * e1) * (e1 * e1)) * (iz4 * iz);
    for (int k = 0; k < 3; ++k) {
      qs[(size_t)k * N] = d1[(size_t)k * N] + d3[(size_t)k * N];
      qd[(size_t)k * N] = d1[(size_t)k * N] - d3[(size_t)k * N];
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Group-gradient pass: d_g (dn/df), the permittivity gradient of each mode's frequency derivative, from the dispersion pass's
// correction x (oracle/mode_group_gradient.py is the float64 model).  With p = (exx, eyy, iez) of the solver frame,
// D_a(w, e) = w^T (dA/dp_a(g)) e is a local product, quadratic in the 1-D coefficients and affine in p, and
//   d_g lambda' w^T v = chi_a [D_a(w_hat, v) + D_a(w, x) + D_a'(w, v)] + chi_a' D_a(w, v) - chi_a D_a(w, v) (w_hat^T v + w^T x) / w^T v
// with w_hat = G'J Q v + G J Q'v + G J Q x (l' = -i Im l for every stretched length), chi = (1/je, 1/je, -iez^2 je),
// chi' = (0, 0, -2 iez iez' je).  Mode 0 sums w_hat^T v per chunk; mode 1 writes
//   map[b][a][g][q] = alpha_b (chi_a E_a + chi_a' D_a) + beta_b chi_a D_a,   E_a = D_a(w_hat, v) + D_a(w, x) + D_a'(w, v),
// with alpha, beta the per-problem scalars of dispersion_pass (NaN for a correction solve that stopped above 100 x inner_tol).
// ------------------------------------------------------------------------------------------------

template <typename T, typename C, bool HAS_MU>
struct GroupCell {
  const T *v, *x;          // this slot's Ritz vector and correction, [e1 | e2]
  const C *fb;             // this problem's coefficient fields: exx, eyy, iez, mxx, myy, imz at fb + k N
  const T *cx, *cy, *dcx, *dcy;  // [4][n] 1-D coefficients and f dc/df
  const cplx *gx, *gy;     // [2][n] primal / dual stretched lengths
  const cplx *p1;          // [3][N] f dp/df, or null
  int nx, ny;
  size_t N;
  __device__ __forceinline__ bool in(int ii, int jj) const { return ii >= 0 && ii < nx && jj >= 0 && jj < ny; }
  __device__ __forceinline__ cplx ld(const T *e, int ii, int jj) const { return in(ii, jj) ? to_cplx(ldg(e + (size_t)ii * ny + jj)) : mk(0.0, 0.0); }
  __device__ __forceinline__ cplx co(const T *c, int n, int w, int i) const { return (i >= 0 && i < n) ? to_cplx(ldg(c + (size_t)w * n + i)) : mk(0.0, 0.0); }
  // 1-D coefficient w of x (ax 0) or y (ax 1) at c + sc c'
  __device__ __forceinline__ cplx cc(int ax, int w, int i, double sc) const {
    cplx c = ax == 0 ? co(cx, nx, w, i) : co(cy, ny, w, i);
    if (sc != 0.0) c += sc * (ax == 0 ? co(dcx, nx, w, i) : co(dcy, ny, w, i));
    return c;
  }
  // coefficient field k (exx, eyy, iez) at (ii, jj) moved by sp p' (zero outside the grid)
  __device__ __forceinline__ cplx fld(int k, int ii, int jj, double sp) const {
    if (!in(ii, jj)) return mk(0.0, 0.0);
    const size_t g = (size_t)ii * ny + jj;
    cplx e = to_cplx(ldg(fb + (size_t)k * N + g));
    if (p1 && sp != 0.0) e += sp * ldg(p1 + (size_t)k * N + g);
    return e;
  }
  __device__ __forceinline__ cplx imz(int ii, int jj) const { return HAS_MU ? to_cplx(ldg(fb + 5 * N + (size_t)ii * ny + jj)) : mk(1.0, 0.0); }
  // t = imz (Dxf e2 - Dyf e1) at (ii, jj) and, with D, its coefficient derivative dt
  template <bool D>
  __device__ __forceinline__ void tt(const T *e, int ii, int jj, cplx &t, cplx &dt) const {
    t = dt = mk(0.0, 0.0);
    if (!in(ii, jj)) return;
    const cplx a2 = ld(e + N, ii, jj), b2 = ld(e + N, ii + 1, jj), a1 = ld(e, ii, jj), b1 = ld(e, ii, jj + 1);
    const cplx mz = imz(ii, jj);
    t = mz * (co(cx, nx, 0, ii) * a2 + co(cx, nx, 1, ii) * b2 - co(cy, ny, 0, jj) * a1 - co(cy, ny, 1, jj) * b1);
    if (D) dt = mz * (co(dcx, nx, 0, ii) * a2 + co(dcx, nx, 1, ii) * b2 - co(dcy, ny, 0, jj) * a1 - co(dcy, ny, 1, jj) * b1);
  }
  // w = G J Q v and w_hat = G'J Q v + G J (Q'v + Q x) at (ii, jj); zero outside the grid
  __device__ __forceinline__ void ww(int ii, int jj, cplx w[2], cplx h[2]) const {
    w[0] = w[1] = h[0] = h[1] = mk(0.0, 0.0);
    if (!in(ii, jj)) return;
    cplx t0, d0, tm, dm, tn, dn, u;
    tt<true>(v, ii, jj, t0, d0);
    tt<true>(v, ii - 1, jj, tm, dm);
    tt<true>(v, ii, jj - 1, tn, dn);
    const cplx e1 = ld(v, ii, jj), e2 = ld(v + N, ii, jj), ex = fld(0, ii, jj, 0.0), ey = fld(1, ii, jj, 0.0);
    const cplx cx2 = co(cx, nx, 2, ii), cx3 = co(cx, nx, 3, ii), cy2 = co(cy, ny, 2, jj), cy3 = co(cy, ny, 3, jj);
    const cplx q1 = cx2 * t0 + cx3 * tm + ey * e2, q2 = cy2 * t0 + cy3 * tn - ex * e1;
    cplx dq1 = co(dcx, nx, 2, ii) * t0 + cx2 * d0 + co(dcx, nx, 3, ii) * tm + cx3 * dm;
    cplx dq2 = co(dcy, ny, 2, jj) * t0 + cy2 * d0 + co(dcy, ny, 3, jj) * tn + cy3 * dn;
    if (p1) {
      const size_t g = (size_t)ii * ny + jj;
      dq1 += ldg(p1 + N + g) * e2;
      dq2 -= ldg(p1 + g) * e1;
    }
    tt<false>(x, ii, jj, t0, u);
    tt<false>(x, ii - 1, jj, tm, u);
    tt<false>(x, ii, jj - 1, tn, u);
    dq1 += cx2 * t0 + cx3 * tm + ey * ld(x + N, ii, jj);
    dq2 += cy2 * t0 + cy3 * tn - ex * ld(x, ii, jj);
    const cplx lfx = gx[ii], lbx = gx[nx + ii], lfy = gy[jj], lby = gy[ny + jj];
    const cplx Gf = lfx * lby, Gb = lbx * lfy;
    const cplx dGf = mk(0.0, -lfx.im) * lby + lfx * mk(0.0, -lby.im), dGb = mk(0.0, -lbx.im) * lfy + lbx * mk(0.0, -lfy.im);
    w[0] = Gf * q2;
    w[1] = -(Gb * q1);
    h[0] = dGf * q2 + Gf * dq2;
    h[1] = -(dGb * q1 + Gb * dq1);
  }
  // D_a(W, e) at (i, j) with coefficients c + sc c' and fields p + sp p'; W: w at (i,j), (i-1,j), (i,j-1), (i+1,j), (i+1,j-1),
  // (i,j+1), (i-1,j+1)
  __device__ __forceinline__ void forms(int i, int j, const cplx (&W)[7][2], const T *e, double sc, double sp, cplx d[3]) const {
    cplx z[3] = {mk(0.0, 0.0), mk(0.0, 0.0), mk(0.0, 0.0)};
#pragma unroll
    for (int s = 0; s < 7; ++s) zadd(s, i, j, W[s][0], W[s][1], sc, z);
    forms_z(i, j, z, W[0][0], W[0][1], e, sc, sp, d);
  }
  // z = Dxf^T w1 + Dyf^T w2 at (i, j), (i+1, j), (i, j+1) with coefficients c + sc c': the part of stencil site s (numbered as
  // for forms) holding w = (w1, w2)
  __device__ __forceinline__ void zadd(int s, int i, int j, cplx w1, cplx w2, double sc, cplx z[3]) const {
    switch (s) {
      case 0:
        z[0] += cc(0, 0, i, sc) * w1 + cc(1, 0, j, sc) * w2;
        if (in(i + 1, j)) z[1] += cc(0, 1, i, sc) * w1;
        if (in(i, j + 1)) z[2] += cc(1, 1, j, sc) * w2;
        break;
      case 1: z[0] += cc(0, 1, i - 1, sc) * w1; break;
      case 2: z[0] += cc(1, 1, j - 1, sc) * w2; break;
      case 3: z[1] += cc(0, 0, i + 1, sc) * w1 + cc(1, 0, j, sc) * w2; break;
      case 4: z[1] += cc(1, 1, j - 1, sc) * w2; break;
      case 5: z[2] += cc(0, 0, i, sc) * w1 + cc(1, 0, j + 1, sc) * w2; break;
      default: z[2] += cc(0, 1, i - 1, sc) * w1; break;
    }
  }
  // D_a from z at (i, j), (i+1, j), (i, j+1) and w at (i, j)
  __device__ __forceinline__ void forms_z(int i, int j, const cplx z[3], cplx w01, cplx w02, const T *e, double sc, double sp, cplx d[3]) const {
    const size_t g = (size_t)i * ny + j;
    const cplx zg = z[0], zx = z[1], zy = z[2];
    const cplx e1 = ld(e, i, j), e2 = ld(e + N, i, j), iz = fld(2, i, j, sp);
    const cplx mx = HAS_MU ? to_cplx(ldg(fb + 3 * N + g)) : mk(1.0, 0.0), my = HAS_MU ? to_cplx(ldg(fb + 4 * N + g)) : mk(1.0, 0.0);
    d[0] = -(e1 * (cc(0, 2, i, sc) * iz * zg + cc(0, 3, i + 1, sc) * fld(2, i + 1, j, sp) * zx + my * w01));
    d[1] = -(e2 * (cc(1, 2, j, sc) * iz * zg + cc(1, 3, j + 1, sc) * fld(2, i, j + 1, sp) * zy + mx * w02));
    const cplx s = cc(0, 2, i, sc) * (fld(0, i, j, sp) * e1) + cc(0, 3, i, sc) * (fld(0, i - 1, j, sp) * ld(e, i - 1, j)) +
                   cc(1, 2, j, sc) * (fld(1, i, j, sp) * e2) + cc(1, 3, j, sc) * (fld(1, i, j - 1, sp) * ld(e + N, i, j - 1));
    d[2] = -(zg * s);
  }
};

// grid (nchunk, B) x 256 threads (mode 0) or like deriv_map_kernel for one mode slot (mode 1), see above.  ab: [B][2] (alpha,
// beta); map: [B][3][N][M].  PERT (mode 1 only): instead of the map, the block sums of (chi E + chi' D, chi D) against the
// perturbations of p (pert_site_sums, NF = 2); the host applies alpha and beta.
template <typename T, typename C, bool HAS_MU, bool PERT = false>
__global__ void __launch_bounds__(256) group_grad_kernel(DispArgs<T, C> a, int mode, const cplx *ab, cplx *map, PertArgs p = PertArgs{}) {
  const DerivArgs<T, C> &d = a.d;
  const int nx = d.nx, ny = d.ny, M = d.num_modes;
  const size_t N = (size_t)nx * ny;
  const int b = mode == 0 ? blockIdx.y : blockIdx.z;
  const T *vb = d.vec + (size_t)a.q * d.vstride + (size_t)b * 2 * N;
  const GroupCell<T, C, HAS_MU> G{vb, a.x + (size_t)b * 2 * N, d.fields + d.field_bstride * b,
                                  d.cx + (size_t)b * 4 * nx, d.cy + (size_t)b * 4 * ny, d.dcx + (size_t)b * 4 * nx, d.dcy + (size_t)b * 4 * ny,
                                  d.gx + (size_t)b * 2 * nx, d.gy + (size_t)b * 2 * ny, a.p1 ? a.p1 + (size_t)b * 3 * N : nullptr, nx, ny, N};
  if (mode == 0) {
    cplx s = mk(0.0, 0.0);
    for (size_t g = (size_t)blockIdx.x * 256 + threadIdx.x; g < N; g += (size_t)gridDim.x * 256) {
      const int i = (int)(g / ny), j = (int)(g % ny);
      cplx w[2], h[2];
      G.ww(i, j, w, h);
      s += h[0] * G.ld(vb, i, j) + h[1] * G.ld(vb + N, i, j);
    }
    __shared__ cplx red[256];
    red[threadIdx.x] = s;
    __syncthreads();
    for (int hh = 128; hh > 0; hh >>= 1) {
      if ((int)threadIdx.x < hh) red[threadIdx.x] += red[threadIdx.x + hh];
      __syncthreads();
    }
    if (threadIdx.x < 3) a.partial[((size_t)b * gridDim.x + blockIdx.x) * 3 + threadIdx.x] = threadIdx.x == 0 ? red[0] : mk(0.0, 0.0);
    return;
  }
  const int j0 = blockIdx.x * 64 + threadIdx.x, i0 = blockIdx.y * 4 + threadIdx.y;
  const bool live = i0 < nx && j0 < ny;
  if (!PERT && !live) return;
  const int i = PERT ? min(i0, nx - 1) : i0, j = PERT ? min(j0, ny - 1) : j0;  // PERT: every thread joins the block sums
  const int di[7] = {0, -1, 0, 1, 1, 0, -1}, dj[7] = {0, 0, -1, 0, -1, 1, 1};
  // D_a(w_hat, v) streams over the stencil (only z and w_hat(i, j) are kept); then the w stencil is kept for the other forms
  cplx W[7][2], un[2], hz[3] = {mk(0.0, 0.0), mk(0.0, 0.0), mk(0.0, 0.0)}, h0[2];
#pragma unroll
  for (int s = 0; s < 7; ++s) {
    cplx hs[2];
    G.ww(i + di[s], j + dj[s], un, hs);
    G.zadd(s, i, j, hs[0], hs[1], 0.0, hz);
    if (s == 0) h0[0] = hs[0], h0[1] = hs[1];
  }
  cplx d0[3], e[3], t[3];
  G.forms_z(i, j, hz, h0[0], h0[1], vb, 0.0, 0.0, e);
#pragma unroll
  for (int s = 0; s < 7; ++s) G.ww(i + di[s], j + dj[s], W[s], un);
  G.forms(i, j, W, vb, 0.0, 0.0, d0);
  G.forms(i, j, W, G.x, 0.0, 0.0, t);
  for (int k = 0; k < 3; ++k) e[k] += t[k];
#pragma unroll 1
  for (int s = 0; s < (a.p1 ? 4 : 2); ++s) {  // D_a'(w, v): +-c', then +-p'
    const double st = (s & 1) ? -0.5 : 0.5;
    G.forms(i, j, W, vb, s < 2 ? 2.0 * st : 0.0, s < 2 ? 0.0 : 2.0 * st, t);
    for (int k = 0; k < 3; ++k) e[k] += st * t[k];
  }
  const size_t g = (size_t)i * ny + j;
  const cplx iz = to_cplx(ldg(G.fb + 2 * N + g));
  const double je = d.jz_e ? d.jz_e[(size_t)b * d.jz_len + (d.jz_axis == 0 ? i : j)] : 1.0;
  const cplx chi[3] = {mk(1.0 / je, 0.0), mk(1.0 / je, 0.0), -(iz * iz) * je};
  const cplx chi1 = a.p1 ? -2.0 * je * (iz * ldg(a.p1 + (size_t)b * 3 * N + 2 * N + g)) : mk(0.0, 0.0);
  const double pec = 0.9 * 1e8;  // PEC-valued input, as eps_grad
  const bool is_pec[3] = {abs2(to_cplx(ldg(G.fb + g))) >= pec * pec, abs2(to_cplx(ldg(G.fb + N + g))) >= pec * pec, abs2(iz) * pec * pec <= 1.0};
  if constexpr (PERT) {
    cplx f[2][3];
    for (int k = 0; k < 3; ++k) {
      f[0][k] = chi[k] * e[k];
      f[1][k] = chi[k] * d0[k];
      if (k == 2) f[0][k] += chi1 * d0[k];
      if (is_pec[k]) f[0][k] = f[1][k] = mk(0.0, 0.0);
    }
    pert_site_sums<2>(p, b, g, N, live, f);
  } else {
    const cplx al = ab[2 * b], be = ab[2 * b + 1];
    cplx *o = map + (size_t)b * 3 * N * M;
    for (int k = 0; k < 3; ++k) {
      cplx num = chi[k] * e[k], g0 = chi[k] * d0[k];
      if (k == 2) num += chi1 * d0[k];
      if (is_pec[k]) num = g0 = mk(0.0, 0.0);
      o[((size_t)k * N + g) * M + a.q] = al * num + be * g0;
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Third-order pass: the third frequency derivative of lambda from the dispersion pass's correction x and the left correction
// w_hat of the group-gradient pass (oracle/mode_third_order.py is the float64 model).  By Wigner's 2n+1 rule,
//   lambda''' w^T v = w^T A'''v + 3 w_hat^T A''v + 3 w^T A''x + 6 w_hat^T A'x - 6 lambda' w_hat^T x - 3 lambda'' (w_hat^T v + w^T x)
// needs no further solve.  A has bidegree (2, 2) in (c, p), so with E(a, b) = A(c + a, p + b) v the terms of A'''v are exact
// with unit steps: A_c[c'''] = [E(c''') - E(-c''')]/2, 3 A_cc[c', c''] = 3/4 [E(c'+c'') - E(c'-c'') - E(-c'+c'') + E(-c'-c'')]
// (A_p, A_pp alike), 3 A_cp[a, b] = 3/4 [E(a, b) - E(a, -b) - E(-a, b) + E(-a, -b)] for (c', p'') and (c'', p'), and
// 3 A_ccp[c', c', p'] + 3 A_cpp[c', p', p'] = 3 [E(c', p') - E(-c', -p') - E(0, p') + E(0, -p') - E(c', 0) + E(-c', 0)].
// Per mode slot one scan sums, per problem, (w_hat^T v, w_hat^T x, w^T A'''v) and (w_hat^T A''v, w^T A''x, w_hat^T A'x).
// ------------------------------------------------------------------------------------------------

// one operator evaluation of A'''v: coefficient direction (0 none, 1 c', 2 c'', 3 c''', 4 c' + c'', 5 c' - c'') and step, field
// direction (0 none, 1 p', 2 p'', 3 p''', 4 p' + p'', 5 p' - p'') and step, weight.  The first six move only the coefficients.
struct ThirdTerm {
  int cdir, pdir;
  double sc, sp, w;
};
__constant__ ThirdTerm kThirdTerms[26] = {
    {3, 0, 1.0, 0.0, 0.5},    {3, 0, -1.0, 0.0, -0.5},  {4, 0, 1.0, 0.0, 0.75},   {5, 0, 1.0, 0.0, -0.75},  {5, 0, -1.0, 0.0, -0.75},
    {4, 0, -1.0, 0.0, 0.75},  {0, 3, 0.0, 1.0, 0.5},    {0, 3, 0.0, -1.0, -0.5},  {0, 4, 0.0, 1.0, 0.75},   {0, 5, 0.0, 1.0, -0.75},
    {0, 5, 0.0, -1.0, -0.75}, {0, 4, 0.0, -1.0, 0.75},  {1, 2, 1.0, 1.0, 0.75},   {1, 2, 1.0, -1.0, -0.75}, {1, 2, -1.0, 1.0, -0.75},
    {1, 2, -1.0, -1.0, 0.75}, {2, 1, 1.0, 1.0, 0.75},   {2, 1, 1.0, -1.0, -0.75}, {2, 1, -1.0, 1.0, -0.75}, {2, 1, -1.0, -1.0, 0.75},
    {1, 1, 1.0, 1.0, 3.0},    {1, 1, -1.0, -1.0, -3.0}, {0, 1, 0.0, 1.0, -3.0},   {0, 1, 0.0, -1.0, 3.0},   {1, 0, 1.0, 0.0, -3.0},
    {1, 0, -1.0, 0.0, 3.0}};

template <typename T>
struct ThirdArgs {
  const T *c3x, *c3y;        // [B][4][n] f^3 d^3c/df^3 = 6 c'^3 / c^2
  const T *csx, *csy;        // [B][4][n] c' + c''
  const T *cdx, *cdy;        // [B][4][n] c' - c''
  const cplx *p3, *ps, *pd;  // [B][3][N] p''', p' + p'', p' - p'' (null with a nondispersive batch)
  cplx *partial;             // [B][2][nchunk][3]
};

// grid (nchunk, B), 256 threads, one mode slot a.q while a.x holds its correction (see above)
template <typename T, typename C, bool HAS_MU>
__global__ void __launch_bounds__(256) third_scan_kernel(DispArgs<T, C> a, ThirdArgs<T> t) {
  const DerivArgs<T, C> &d = a.d;
  const int b = blockIdx.y, nx = d.nx, ny = d.ny;
  const size_t N = (size_t)nx * ny;
  const bool hp = a.p1 != nullptr;
  const DispTerm *tab2 = hp ? kDispTermsP : kDispTermsC;
  const int n2 = hp ? 13 : 5, n3 = hp ? 26 : 6;
  const T *vb = d.vec + (size_t)a.q * d.vstride + (size_t)b * 2 * N, *xb = a.x + (size_t)b * 2 * N;
  const size_t o4x = (size_t)b * 4 * nx, o4y = (size_t)b * 4 * ny, o3 = (size_t)b * 3 * N;
  const GroupCell<T, C, HAS_MU> G{vb, xb, d.fields + d.field_bstride * b, d.cx + o4x, d.cy + o4y, d.dcx + o4x, d.dcy + o4y,
                                  d.gx + (size_t)b * 2 * nx, d.gy + (size_t)b * 2 * ny, hp ? a.p1 + o3 : nullptr, nx, ny, N};
  const T *cxb = d.cx + o4x, *cyb = d.cy + o4y;
  // direction k of the coefficients (per axis) and of the fields, selected per term (a table of pointers would stay in registers)
  auto rows = [&](int k, int ax) -> const T * {
    const size_t o = ax == 0 ? o4x : o4y;
    switch (k) {
      case 1: return (ax == 0 ? d.dcx : d.dcy) + o;
      case 2: return (ax == 0 ? a.c2x : a.c2y) + o;
      case 3: return (ax == 0 ? t.c3x : t.c3y) + o;
      case 4: return (ax == 0 ? t.csx : t.csy) + o;
      case 5: return (ax == 0 ? t.cdx : t.cdy) + o;
      default: return nullptr;
    }
  };
  auto fdir = [&](int k) -> const cplx * {
    if (!hp) return nullptr;
    switch (k) {
      case 1: return a.p1 + o3;
      case 2: return a.p2 + o3;
      case 3: return t.p3 + o3;
      case 4: return t.ps + o3;
      case 5: return t.pd + o3;
      default: return nullptr;
    }
  };
  const C *fb = d.fields + d.field_bstride * b;
  cplx s[6] = {mk(0.0, 0.0), mk(0.0, 0.0), mk(0.0, 0.0), mk(0.0, 0.0), mk(0.0, 0.0), mk(0.0, 0.0)};
  for (size_t g = (size_t)blockIdx.x * 256 + threadIdx.x; g < N; g += (size_t)gridDim.x * 256) {
    const int i = (int)(g / ny), j = (int)(g % ny);
    cplx a2v[2] = {mk(0.0, 0.0), mk(0.0, 0.0)}, a2x[2] = {mk(0.0, 0.0), mk(0.0, 0.0)}, a1x[2] = {mk(0.0, 0.0), mk(0.0, 0.0)};
#pragma unroll 1
    for (int k = 0; k < n2; ++k) {  // A'' on v and on x, A' on x
      const DispTerm tm = tab2[k];
      const CoefRows<T> CX{cxb, rows(tm.cdir, 0), tm.sc, nx}, CY{cyb, rows(tm.cdir, 1), tm.sc, ny};
      const cplx *dp = fdir(tm.pdir);
      const PertSite<T, C, HAS_MU> Pv{vb, vb + N, fb, dp, tm.sp, CX, CY, nx, ny, N};
      const PertSite<T, C, HAS_MU> Px{xb, xb + N, fb, dp, tm.sp, CX, CY, nx, ny, N};
      cplx y1, y2;
      Pv.apply(i, j, y1, y2);
      a2v[0] += tm.w2 * y1;
      a2v[1] += tm.w2 * y2;
      Px.apply(i, j, y1, y2);
      a2x[0] += tm.w2 * y1;
      a2x[1] += tm.w2 * y2;
      a1x[0] += tm.w1 * y1;
      a1x[1] += tm.w1 * y2;
    }
    cplx a3v[2] = {mk(0.0, 0.0), mk(0.0, 0.0)};
#pragma unroll 1
    for (int k = 0; k < n3; ++k) {  // A''' on v
      const ThirdTerm tm = kThirdTerms[k];
      const PertSite<T, C, HAS_MU> Pv{vb, vb + N, fb, fdir(tm.pdir), tm.sp, CoefRows<T>{cxb, rows(tm.cdir, 0), tm.sc, nx},
                                      CoefRows<T>{cyb, rows(tm.cdir, 1), tm.sc, ny}, nx, ny, N};
      cplx y1, y2;
      Pv.apply(i, j, y1, y2);
      a3v[0] += tm.w * y1;
      a3v[1] += tm.w * y2;
    }
    cplx w[2], h[2];  // w and w_hat at (i, j), formed after the operator terms so that they do not hold registers through them
    G.ww(i, j, w, h);
    s[0] += h[0] * to_cplx(ldg(vb + g)) + h[1] * to_cplx(ldg(vb + N + g));
    s[1] += h[0] * to_cplx(ldg(xb + g)) + h[1] * to_cplx(ldg(xb + N + g));
    s[2] += w[0] * a3v[0] + w[1] * a3v[1];
    s[3] += h[0] * a2v[0] + h[1] * a2v[1];
    s[4] += w[0] * a2x[0] + w[1] * a2x[1];
    s[5] += h[0] * a1x[0] + h[1] * a1x[1];
  }
  __shared__ cplx red[6][256];
  for (int k = 0; k < 6; ++k) red[k][threadIdx.x] = s[k];
  __syncthreads();
  for (int hh = 128; hh > 0; hh >>= 1) {
    if ((int)threadIdx.x < hh)
      for (int k = 0; k < 6; ++k) red[k][threadIdx.x] += red[k][threadIdx.x + hh];
    __syncthreads();
  }
  if (threadIdx.x < 6) t.partial[(((size_t)b * 2 + threadIdx.x / 3) * gridDim.x + blockIdx.x) * 3 + threadIdx.x % 3] = red[threadIdx.x][0];
}

// ------------------------------------------------------------------------------------------------
// Fourth-order pass: the fourth frequency derivative of lambda from a second-order right correction x2 and the structural
// second-order left correction w_hat2 (oracle/mode_fourth_order.py is the float64 model).  Per mode slot, after every stage of
// the slot that reads x: fourth_rhs_kernel writes r2 = -[(A' - lambda') x + (A'' - lambda'') v / 2] (w^T r2 = 0 is the formula
// for lambda''), the eigen-solve's inner solver gives (A - lambda) x2 = r2, and fourth_scan_kernel sums (PART 0)
//   w^T (A''''v + 4 A'''x),  w_hat^T A'''v
// and (PART 1)
//   w_hat2^T (12 A''v + 24 A'x + 24 (A - lambda) x2),  w^T A''x2,  w_hat^T (12 A''x + 24 A'x2),  w_hat2^T v,  w^T x2,  w_hat2^T x,
//   w_hat^T x2,
// from which the host forms
//   lambda'''' w^T v = [the five products] - 24 lambda' D_3 - 12 lambda'' D_2 - 4 lambda''' D_1
// (D_k: the t^k coefficient of (w + t w_hat + t^2 w_hat2)^T (v + t x + t^2 x2)).  A''''v is exact from the 64 unit-step
// evaluations of kFourthTerms (the first nine move only the coefficients; their derivation is in fourth_operator of the model).
// w_hat2 = G_2 J Q v + G_1 J (Q_1 v + Q x) + G J (Q_2 v + Q_1 x + Q x2) is formed per cell like w_hat (SecondCell::ww2).
// ------------------------------------------------------------------------------------------------

// one operator evaluation of A''''v, in the direction numbering of ThirdTerm extended by 6 c'''' (p''''), 7 c' + c''' (p' + p''')
// and 8 c' - c''' (p' - p''')
__constant__ ThirdTerm kFourthTerms[64] = {
    {6, 0, 1.0, 0.0, 0.5}, {6, 0, -1.0, 0.0, -0.5}, {7, 0, 1.0, 0.0, 1}, {8, 0, 1.0, 0.0, -1}, {8, 0, -1.0, 0.0, -1},
    {7, 0, -1.0, 0.0, 1}, {2, 0, 1.0, 0.0, 3}, {2, 0, -1.0, 0.0, 3}, {0, 0, 0.0, 0.0, -6}, {2, 0, 1.0, 0.0, -6},
    {2, 0, -1.0, 0.0, 6}, {0, 0, 0.0, 0.0, 18}, {0, 6, 0.0, 1.0, 0.5}, {0, 6, 0.0, -1.0, -0.5}, {0, 7, 0.0, 1.0, 1},
    {0, 8, 0.0, 1.0, -1}, {0, 8, 0.0, -1.0, -1}, {0, 7, 0.0, -1.0, 1}, {0, 2, 0.0, 1.0, -3}, {0, 2, 0.0, -1.0, 9},
    {1, 3, 1.0, 1.0, 1}, {1, 3, 1.0, -1.0, -1}, {1, 3, -1.0, 1.0, -1}, {1, 3, -1.0, -1.0, 1}, {2, 2, 1.0, 1.0, 1.5},
    {2, 2, 1.0, -1.0, -1.5}, {2, 2, -1.0, 1.0, -1.5}, {2, 2, -1.0, -1.0, 1.5}, {3, 1, 1.0, 1.0, 1}, {3, 1, 1.0, -1.0, -1},
    {3, 1, -1.0, 1.0, -1}, {3, 1, -1.0, -1.0, 1}, {1, 2, 1.0, 1.0, 3}, {1, 2, 1.0, -1.0, -3}, {1, 2, -1.0, 1.0, 3},
    {1, 2, -1.0, -1.0, -3}, {4, 1, 1.0, 1.0, 1.5}, {4, 1, 1.0, -1.0, -1.5}, {4, 1, -1.0, 1.0, 1.5}, {4, 1, -1.0, -1.0, -1.5},
    {5, 1, 1.0, 1.0, -1.5}, {5, 1, 1.0, -1.0, 1.5}, {5, 1, -1.0, 1.0, -1.5}, {5, 1, -1.0, -1.0, 1.5}, {2, 1, 1.0, 1.0, 3},
    {2, 1, 1.0, -1.0, 3}, {2, 1, -1.0, 1.0, -3}, {2, 1, -1.0, -1.0, -3}, {1, 4, 1.0, 1.0, 1.5}, {1, 4, 1.0, -1.0, 1.5},
    {1, 4, -1.0, 1.0, -1.5}, {1, 4, -1.0, -1.0, -1.5}, {1, 5, 1.0, 1.0, -1.5}, {1, 5, 1.0, -1.0, -1.5}, {1, 5, -1.0, 1.0, 1.5},
    {1, 5, -1.0, -1.0, 1.5}, {1, 1, 1.0, 1.0, 6}, {1, 1, 1.0, -1.0, 6}, {1, 1, -1.0, 1.0, 6}, {1, 1, -1.0, -1.0, 6},
    {1, 0, 1.0, 0.0, -12}, {1, 0, -1.0, 0.0, -12}, {0, 1, 0.0, 1.0, -12}, {0, 1, 0.0, -1.0, -12}};

template <typename T>
struct FourthArgs {
  const T *c4x, *c4y;          // [B][4][n] f^4 d^4c/df^4 = 24 c'^4 / c^3
  const T *qsx, *qsy;          // [B][4][n] c' + c'''
  const T *qdx, *qdy;          // [B][4][n] c' - c'''
  const cplx *p4, *qs, *qd;    // [B][3][N] p'''', p' + p''', p' - p''' (null with a nondispersive batch)
  const T *x2;                 // the second-order correction, batched-vector layout
  const cplx *sc;              // [B][3] lambda', lambda'', lambda (scaled)
  cplx *partial;               // [B][4][nchunk][3]
};

// grid (min(N/256, 1024), B), 256 threads: r2 of mode slot a.q into `r2` while a.x holds its first-order correction
template <typename T, typename C, bool HAS_MU>
__global__ void __launch_bounds__(256) fourth_rhs_kernel(DispArgs<T, C> a, const cplx *sc, T *r2) {
  const int b = blockIdx.y, nx = a.d.nx, ny = a.d.ny;
  const size_t N = (size_t)nx * ny;
  const bool hp = a.p1 != nullptr;
  const DispTerm *tab = hp ? kDispTermsP : kDispTermsC;
  const int nterm = hp ? 13 : 5;
  const T *vb = a.d.vec + (size_t)a.q * a.d.vstride + (size_t)b * 2 * N, *xb = a.x + (size_t)b * 2 * N;
  const T *cxb = a.d.cx + (size_t)b * 4 * nx, *cyb = a.d.cy + (size_t)b * 4 * ny;
  const T *d1x = a.d.dcx + (size_t)b * 4 * nx, *d1y = a.d.dcy + (size_t)b * 4 * ny;
  const T *d2x = a.c2x + (size_t)b * 4 * nx, *d2y = a.c2y + (size_t)b * 4 * ny;
  const cplx *p1 = hp ? a.p1 + (size_t)b * 3 * N : nullptr, *p2 = hp ? a.p2 + (size_t)b * 3 * N : nullptr;
  const C *fb = a.d.fields + a.d.field_bstride * b;
  const cplx l1 = sc[3 * b], l2 = sc[3 * b + 1];
  T *rb = r2 + (size_t)b * 2 * N;
  for (size_t g = (size_t)blockIdx.x * 256 + threadIdx.x; g < N; g += (size_t)gridDim.x * 256) {
    const int i = (int)(g / ny), j = (int)(g % ny);
    cplx y[2] = {mk(0.0, 0.0), mk(0.0, 0.0)};  // (A' - lambda') x + (A'' - lambda'') v / 2, without the lambda terms
#pragma unroll 1
    for (int t = 0; t < nterm; ++t) {
      const DispTerm tm = tab[t];
      const T *dcx = tm.cdir == 1 ? d1x : (tm.cdir == 2 ? d2x : nullptr), *dcy = tm.cdir == 1 ? d1y : (tm.cdir == 2 ? d2y : nullptr);
      const cplx *dp = tm.pdir == 1 ? p1 : (tm.pdir == 2 ? p2 : nullptr);
      const CoefRows<T> CX{cxb, dcx, tm.sc, nx}, CY{cyb, dcy, tm.sc, ny};
      const PertSite<T, C, HAS_MU> Pv{vb, vb + N, fb, dp, tm.sp, CX, CY, nx, ny, N}, Px{xb, xb + N, fb, dp, tm.sp, CX, CY, nx, ny, N};
      cplx y1, y2;
      Pv.apply(i, j, y1, y2);
      y[0] += (0.5 * tm.w2) * y1;
      y[1] += (0.5 * tm.w2) * y2;
      Px.apply(i, j, y1, y2);
      y[0] += tm.w1 * y1;
      y[1] += tm.w1 * y2;
    }
    for (int c = 0; c < 2; ++c) {
      const cplx e = to_cplx(ldg(vb + (size_t)c * N + g)), x = to_cplx(ldg(xb + (size_t)c * N + g));
      rb[(size_t)c * N + g] = cast_to<T>(-(y[c] - l1 * x - (0.5 * l2) * e));
    }
  }
}

// w, w_hat and w_hat2 of one mode slot at a cell: GroupCell (v, x, c', p') with x2, c'' and p''
template <typename T, typename C, bool HAS_MU>
struct SecondCell {
  GroupCell<T, C, HAS_MU> G;
  const T *x2;
  const T *c2x, *c2y;  // [4][n] f^2 d^2c/df^2 of this problem
  const cplx *p2;      // [3][N] f^2 d^2p/df^2, or null
  // t = imz (Dxf e2 - Dyf e1) at (ii, jj) with the 1-D coefficient rows ax, ay (zero outside the grid)
  __device__ __forceinline__ cplx t(const T *e, int ii, int jj, const T *ax, const T *ay) const {
    if (!G.in(ii, jj)) return mk(0.0, 0.0);
    const int nx = G.nx, ny = G.ny;
    const size_t N = G.N;
    return G.imz(ii, jj) * (G.co(ax, nx, 0, ii) * G.ld(e + N, ii, jj) + G.co(ax, nx, 1, ii) * G.ld(e + N, ii + 1, jj) -
                            G.co(ay, ny, 0, jj) * G.ld(e, ii, jj) - G.co(ay, ny, 1, jj) * G.ld(e, ii, jj + 1));
  }
  // (q1, q2) of Q e at (ii, jj): backward rows bx, by applied to the t of the forward rows fx, fy, plus the eps term of `fld`
  // (k-th field of a [3][N] direction, or the coefficient fields for fld == null) scaled by s
  __device__ __forceinline__ void q(const T *e, int ii, int jj, const T *bx, const T *by, const T *fx, const T *fy, const cplx *fld,
                                    double s, cplx &q1, cplx &q2) const {
    const int nx = G.nx, ny = G.ny;
    const size_t g = (size_t)ii * ny + jj;
    q1 = mk(0.0, 0.0);
    q2 = mk(0.0, 0.0);
    if (bx) {
      const cplx t0 = t(e, ii, jj, fx, fy);
      q1 = G.co(bx, nx, 2, ii) * t0 + G.co(bx, nx, 3, ii) * t(e, ii - 1, jj, fx, fy);
      q2 = G.co(by, ny, 2, jj) * t0 + G.co(by, ny, 3, jj) * t(e, ii, jj - 1, fx, fy);
    }
    if (s != 0.0) {
      const cplx ex = fld ? ldg(fld + g) : to_cplx(ldg(G.fb + g)), ey = fld ? ldg(fld + G.N + g) : to_cplx(ldg(G.fb + G.N + g));
      q1 += (s * ey) * G.ld(e + G.N, ii, jj);
      q2 -= (s * ex) * G.ld(e, ii, jj);
    }
  }
  __device__ __forceinline__ void ww2(int ii, int jj, cplx w[2], cplx h[2], cplx h2[2]) const {
    w[0] = w[1] = h[0] = h[1] = h2[0] = h2[1] = mk(0.0, 0.0);
    if (!G.in(ii, jj)) return;
    const T *v = G.v, *x = G.x;
    const cplx *c = nullptr;  // no eps term
    const T *cx = G.cx, *cy = G.cy, *dx = G.dcx, *dy = G.dcy, *ex = c2x, *ey = c2y;
    cplx a1, a2, b1, b2;
    cplx q01, q02;  // Q v
    q(v, ii, jj, cx, cy, cx, cy, nullptr, 1.0, q01, q02);
    cplx q11 = mk(0.0, 0.0), q12 = mk(0.0, 0.0);  // Q_1 v + Q x
    q(v, ii, jj, dx, dy, cx, cy, c, 0.0, a1, a2);
    q(v, ii, jj, cx, cy, dx, dy, G.p1, G.p1 ? 1.0 : 0.0, b1, b2);
    q11 = a1 + b1;
    q12 = a2 + b2;
    q(x, ii, jj, cx, cy, cx, cy, nullptr, 1.0, a1, a2);
    q11 += a1;
    q12 += a2;
    // Q_2 v + Q_1 x + Q x2, Q_2 v = B(c', c') v + Q_c[c''/2] v + Q_p[p''/2] v
    cplx q21, q22;
    q(v, ii, jj, dx, dy, dx, dy, p2, p2 ? 0.5 : 0.0, q21, q22);
    q(v, ii, jj, ex, ey, cx, cy, c, 0.0, a1, a2);
    q(v, ii, jj, cx, cy, ex, ey, c, 0.0, b1, b2);
    q21 += 0.5 * (a1 + b1);
    q22 += 0.5 * (a2 + b2);
    q(x, ii, jj, dx, dy, cx, cy, c, 0.0, a1, a2);
    q(x, ii, jj, cx, cy, dx, dy, G.p1, G.p1 ? 1.0 : 0.0, b1, b2);
    q21 += a1 + b1;
    q22 += a2 + b2;
    q(x2, ii, jj, cx, cy, cx, cy, nullptr, 1.0, a1, a2);
    q21 += a1;
    q22 += a2;
    const int nx = G.nx, ny = G.ny;
    const cplx lfx = G.gx[ii], lbx = G.gx[nx + ii], lfy = G.gy[jj], lby = G.gy[ny + jj];
    auto d1 = [](cplx l) { return mk(0.0, -l.im); };  // l_1 = -i Im l, l_2 = i Im l
    auto d2 = [](cplx l) { return mk(0.0, l.im); };
    const cplx Gf = lfx * lby, Gb = lbx * lfy;
    const cplx dGf = d1(lfx) * lby + lfx * d1(lby), dGb = d1(lbx) * lfy + lbx * d1(lfy);
    const cplx eGf = d2(lfx) * lby + d1(lfx) * d1(lby) + lfx * d2(lby), eGb = d2(lbx) * lfy + d1(lbx) * d1(lfy) + lbx * d2(lfy);
    w[0] = Gf * q02;
    w[1] = -(Gb * q01);
    h[0] = dGf * q02 + Gf * q12;
    h[1] = -(dGb * q01 + Gb * q11);
    h2[0] = eGf * q02 + dGf * q12 + Gf * q22;
    h2[1] = -(eGb * q01 + dGb * q11 + Gb * q21);
  }
};

// grid (nchunk, B), 256 threads, one mode slot a.q while a.x holds its first-order correction and u.x2 its second-order one:
// PART 0 writes group 0 of u.partial, PART 1 groups 1-3 (see above)
template <typename T, typename C, bool HAS_MU, int PART>
__global__ void __launch_bounds__(256) fourth_scan_kernel(DispArgs<T, C> a, ThirdArgs<T> t, FourthArgs<T> u) {
  const DerivArgs<T, C> &d = a.d;
  const int b = blockIdx.y, nx = d.nx, ny = d.ny;
  const size_t N = (size_t)nx * ny;
  const bool hp = a.p1 != nullptr;
  const T *vb = d.vec + (size_t)a.q * d.vstride + (size_t)b * 2 * N, *xb = a.x + (size_t)b * 2 * N, *x2b = u.x2 + (size_t)b * 2 * N;
  const size_t o4x = (size_t)b * 4 * nx, o4y = (size_t)b * 4 * ny, o3 = (size_t)b * 3 * N;
  const GroupCell<T, C, HAS_MU> G{vb, xb, d.fields + d.field_bstride * b, d.cx + o4x, d.cy + o4y, d.dcx + o4x, d.dcy + o4y,
                                  d.gx + (size_t)b * 2 * nx, d.gy + (size_t)b * 2 * ny, hp ? a.p1 + o3 : nullptr, nx, ny, N};
  const T *cxb = d.cx + o4x, *cyb = d.cy + o4y;
  auto rows = [&](int k, int ax) -> const T * {  // as in third_scan_kernel, with 6-8 of kFourthTerms
    const size_t o = ax == 0 ? o4x : o4y;
    switch (k) {
      case 1: return (ax == 0 ? d.dcx : d.dcy) + o;
      case 2: return (ax == 0 ? a.c2x : a.c2y) + o;
      case 3: return (ax == 0 ? t.c3x : t.c3y) + o;
      case 4: return (ax == 0 ? t.csx : t.csy) + o;
      case 5: return (ax == 0 ? t.cdx : t.cdy) + o;
      case 6: return (ax == 0 ? u.c4x : u.c4y) + o;
      case 7: return (ax == 0 ? u.qsx : u.qsy) + o;
      case 8: return (ax == 0 ? u.qdx : u.qdy) + o;
      default: return nullptr;
    }
  };
  auto fdir = [&](int k) -> const cplx * {
    if (!hp) return nullptr;
    switch (k) {
      case 1: return a.p1 + o3;
      case 2: return a.p2 + o3;
      case 3: return t.p3 + o3;
      case 4: return t.ps + o3;
      case 5: return t.pd + o3;
      case 6: return u.p4 + o3;
      case 7: return u.qs + o3;
      case 8: return u.qd + o3;
      default: return nullptr;
    }
  };
  const C *fb = d.fields + d.field_bstride * b;
  cplx s[9];
  for (int k = 0; k < 9; ++k) s[k] = mk(0.0, 0.0);
  for (size_t g = (size_t)blockIdx.x * 256 + threadIdx.x; g < N; g += (size_t)gridDim.x * 256) {
    const int i = (int)(g / ny), j = (int)(g % ny);
    if (PART == 0) {
      cplx yw[2] = {mk(0.0, 0.0), mk(0.0, 0.0)}, yh[2] = {mk(0.0, 0.0), mk(0.0, 0.0)};  // A''''v + 4 A'''x, A'''v
#pragma unroll 1
      for (int k = 0; k < (hp ? 26 : 6); ++k) {
        const ThirdTerm tm = kThirdTerms[k];
        const CoefRows<T> CX{cxb, rows(tm.cdir, 0), tm.sc, nx}, CY{cyb, rows(tm.cdir, 1), tm.sc, ny};
        const cplx *dp = fdir(tm.pdir);
        const PertSite<T, C, HAS_MU> Pv{vb, vb + N, fb, dp, tm.sp, CX, CY, nx, ny, N}, Px{xb, xb + N, fb, dp, tm.sp, CX, CY, nx, ny, N};
        cplx y1, y2;
        Pv.apply(i, j, y1, y2);
        yh[0] += tm.w * y1;
        yh[1] += tm.w * y2;
        Px.apply(i, j, y1, y2);
        yw[0] += (4.0 * tm.w) * y1;
        yw[1] += (4.0 * tm.w) * y2;
      }
#pragma unroll 1
      for (int k = 0; k < (hp ? 64 : 9); ++k) {
        const ThirdTerm tm = kFourthTerms[k];
        const PertSite<T, C, HAS_MU> Pv{vb, vb + N, fb, fdir(tm.pdir), tm.sp, CoefRows<T>{cxb, rows(tm.cdir, 0), tm.sc, nx},
                                        CoefRows<T>{cyb, rows(tm.cdir, 1), tm.sc, ny}, nx, ny, N};
        cplx y1, y2;
        Pv.apply(i, j, y1, y2);
        yw[0] += tm.w * y1;
        yw[1] += tm.w * y2;
      }
      cplx w[2], h[2];
      G.ww(i, j, w, h);
      s[0] += w[0] * yw[0] + w[1] * yw[1];
      s[1] += h[0] * yh[0] + h[1] * yh[1];
    } else {
      const DispTerm *tab2 = hp ? kDispTermsP : kDispTermsC;
      const cplx lam = u.sc[3 * b + 2];
      // A''x2 (w), 12 A''x + 24 A'x2 (w_hat), 12 A''v + 24 A'x + 24 (A - lambda) x2 (w_hat2)
      cplx yw[2] = {mk(0.0, 0.0), mk(0.0, 0.0)}, yh[2] = {mk(0.0, 0.0), mk(0.0, 0.0)}, yh2[2];
      {
        const PertSite<T, C, HAS_MU> P0{x2b, x2b + N, fb, nullptr, 0.0, CoefRows<T>{cxb, nullptr, 0.0, nx}, CoefRows<T>{cyb, nullptr, 0.0, ny},
                                        nx, ny, N};
        cplx y1, y2;
        P0.apply(i, j, y1, y2);
        yh2[0] = 24.0 * (y1 - lam * to_cplx(ldg(x2b + g)));
        yh2[1] = 24.0 * (y2 - lam * to_cplx(ldg(x2b + N + g)));
      }
#pragma unroll 1
      for (int k = 0; k < (hp ? 13 : 5); ++k) {
        const DispTerm tm = tab2[k];
        const CoefRows<T> CX{cxb, rows(tm.cdir, 0), tm.sc, nx}, CY{cyb, rows(tm.cdir, 1), tm.sc, ny};
        const cplx *dp = fdir(tm.pdir);
        const PertSite<T, C, HAS_MU> Pv{vb, vb + N, fb, dp, tm.sp, CX, CY, nx, ny, N}, Px{xb, xb + N, fb, dp, tm.sp, CX, CY, nx, ny, N};
        const PertSite<T, C, HAS_MU> Px2{x2b, x2b + N, fb, dp, tm.sp, CX, CY, nx, ny, N};
        cplx y1, y2;
        Pv.apply(i, j, y1, y2);
        yh2[0] += (12.0 * tm.w2) * y1;
        yh2[1] += (12.0 * tm.w2) * y2;
        Px.apply(i, j, y1, y2);
        yh2[0] += (24.0 * tm.w1) * y1;
        yh2[1] += (24.0 * tm.w1) * y2;
        yh[0] += (12.0 * tm.w2) * y1;
        yh[1] += (12.0 * tm.w2) * y2;
        Px2.apply(i, j, y1, y2);
        yh[0] += (24.0 * tm.w1) * y1;
        yh[1] += (24.0 * tm.w1) * y2;
        yw[0] += tm.w2 * y1;
        yw[1] += tm.w2 * y2;
      }
      const SecondCell<T, C, HAS_MU> S2{G, x2b, a.c2x + o4x, a.c2y + o4y, hp ? a.p2 + o3 : nullptr};
      cplx w[2], h[2], h2[2];
      S2.ww2(i, j, w, h, h2);
      const cplx e1 = to_cplx(ldg(vb + g)), e2 = to_cplx(ldg(vb + N + g)), x1 = to_cplx(ldg(xb + g)), x2 = to_cplx(ldg(xb + N + g));
      const cplx z1 = to_cplx(ldg(x2b + g)), z2 = to_cplx(ldg(x2b + N + g));
      s[2] += h2[0] * yh2[0] + h2[1] * yh2[1];
      s[3] += w[0] * yw[0] + w[1] * yw[1];
      s[4] += h[0] * yh[0] + h[1] * yh[1];
      s[5] += h2[0] * e1 + h2[1] * e2;
      s[6] += w[0] * z1 + w[1] * z2;
      s[7] += h2[0] * x1 + h2[1] * x2;
      s[8] += h[0] * z1 + h[1] * z2;
    }
  }
  // PART 0: slots 0-2 of group 0 hold s[0], s[1], 0; PART 1: groups 1-3 hold s[2..8], 0, 0
  const int lo = PART == 0 ? 0 : 2, nsum = PART == 0 ? 3 : 9;
  __shared__ cplx red[9][256];
#pragma unroll
  for (int k = 0; k < nsum; ++k) red[k][threadIdx.x] = (lo + k <= (PART == 0 ? 1 : 8)) ? s[lo + k] : mk(0.0, 0.0);
  __syncthreads();
  for (int hh = 128; hh > 0; hh >>= 1) {
    if ((int)threadIdx.x < hh)
      for (int k = 0; k < nsum; ++k) red[k][threadIdx.x] += red[k][threadIdx.x + hh];
    __syncthreads();
  }
  const int g0 = PART == 0 ? 0 : 1;
  if ((int)threadIdx.x < nsum)
    u.partial[(((size_t)b * 4 + g0 + threadIdx.x / 3) * gridDim.x + blockIdx.x) * 3 + threadIdx.x % 3] = red[threadIdx.x][0];
}

// ------------------------------------------------------------------------------------------------
// Dispersion-gradient pass: d_g (d^2n/df^2), the permittivity gradient of each mode's second frequency derivative, from the
// corrections x, x2 of the fourth-order pass (oracle/mode_dispersion_gradient.py is the float64 model).  In t = (f_new - f) / f,
// with v(t) = v + t x + t^2 x2 and w(t) = w + t w_hat + t^2 w_hat2, the t^0..t^2 coefficients of N/D are stationary in all six
// vectors, so d_g lambda_2 (lambda_2 = lambda''/2) is [t^2] of E(t) / D(t) at fixed vectors, E(t) = chi_a(t) D_a(t)(w(t), v(t)):
//   E_0 = chi D(w, v),   E_1 = chi [D(w_hat, v) + D(w, x) + D_1(w, v)] + chi_1 D(w, v),
//   E_2 = chi [D(w_hat2, v) + D(w_hat, x) + D(w, x2) + D_1(w_hat, v) + D_1(w, x) + D_2(w, v)] + chi_1 [D(w_hat, v) + D(w, x) + D_1(w, v)]
//         + chi_2 D(w, v),
// D_k the t^k coefficient of the form at (c + t c' + t^2 c''/2, p + t p' + t^2 p''/2): D_1 = [D(c+c') - D(c-c')]/2 + [D(p+p') - D(p-p')]/2,
// D_2 = [D(c+c') + D(c-c')]/2 - D + [D(c+c''/2) - D(c-c''/2)]/2 + [D(p+p''/2) - D(p-p''/2)]/2 + [D(c'+, p'+) - D(c'+, p'-) - D(c'-, p'+)
// + D(c'-, p'-)]/4, all exact with unit steps.  chi_zz(t) = -je iez(t)^2: chi_1 = -2 je iez iez', chi_2 = -je (2 iez iez''/2 + iez'^2).
// The host folds d_g lambda_2 = E_2/D_0 - (E_1 D_1 + E_0 D_2)/D_0^2 + E_0 D_1^2/D_0^3 and the chain to n'' into three scalars per
// problem, so map[b][a][g][q] = beta_0 E_0 + beta_1 E_1 + beta_2 E_2 (NaN where d4n_dfreq4 is NaN).
// ------------------------------------------------------------------------------------------------

// grid like deriv_map_kernel for one mode slot a.q while a.x holds its first-order correction and u.x2 its second-order one;
// beta: [B][3]; map: [B][3][N][M].  PERT: instead of the map, the block sums of (E_0, E_1, E_2) against the perturbations of p
// (pert_site_sums, NF = 3); the host applies beta_0..beta_2.
template <typename T, typename C, bool HAS_MU, bool PERT = false>
__global__ void __launch_bounds__(256) disp_grad_kernel(DispArgs<T, C> a, FourthArgs<T> u, const cplx *beta, cplx *map, PertArgs p = PertArgs{}) {
  const DerivArgs<T, C> &d = a.d;
  const int nx = d.nx, ny = d.ny, M = d.num_modes, b = blockIdx.z;
  const size_t N = (size_t)nx * ny;
  const int j0 = blockIdx.x * 64 + threadIdx.x, i0 = blockIdx.y * 4 + threadIdx.y;
  const bool live = i0 < nx && j0 < ny;
  if (!PERT && !live) return;
  const int i = PERT ? min(i0, nx - 1) : i0, j = PERT ? min(j0, ny - 1) : j0;  // PERT: every thread joins the block sums
  const bool hp = a.p1 != nullptr;
  const T *vb = d.vec + (size_t)a.q * d.vstride + (size_t)b * 2 * N, *xb = a.x + (size_t)b * 2 * N, *x2b = u.x2 + (size_t)b * 2 * N;
  const size_t o4x = (size_t)b * 4 * nx, o4y = (size_t)b * 4 * ny, o3 = (size_t)b * 3 * N;
  const GroupCell<T, C, HAS_MU> G{vb, xb, d.fields + d.field_bstride * b, d.cx + o4x, d.cy + o4y, d.dcx + o4x, d.dcy + o4y,
                                  d.gx + (size_t)b * 2 * nx, d.gy + (size_t)b * 2 * ny, hp ? a.p1 + o3 : nullptr, nx, ny, N};
  GroupCell<T, C, HAS_MU> G2 = G;  // the same site with the directions c'' and p'' in place of c' and p'
  G2.dcx = a.c2x + o4x;
  G2.dcy = a.c2y + o4y;
  G2.p1 = hp ? a.p2 + o3 : nullptr;
  const SecondCell<T, C, HAS_MU> S2{G, x2b, a.c2x + o4x, a.c2y + o4y, hp ? a.p2 + o3 : nullptr};
  const int di[7] = {0, -1, 0, 1, 1, 0, -1}, dj[7] = {0, 0, -1, 0, -1, 1, 1};
  // w_hat and w_hat2 stream over the stencil: z of w_hat at c, c + c', c - c' and of w_hat2 at c, and both at (i, j)
  cplx hz[3][3], h2z[3], h0[2], h20[2], un[2];
  for (int k = 0; k < 3; ++k) hz[0][k] = hz[1][k] = hz[2][k] = h2z[k] = mk(0.0, 0.0);
#pragma unroll
  for (int s = 0; s < 7; ++s) {
    cplx hs[2], h2s[2];
    S2.ww2(i + di[s], j + dj[s], un, hs, h2s);
    G.zadd(s, i, j, hs[0], hs[1], 0.0, hz[0]);
    G.zadd(s, i, j, hs[0], hs[1], 1.0, hz[1]);
    G.zadd(s, i, j, hs[0], hs[1], -1.0, hz[2]);
    G.zadd(s, i, j, h2s[0], h2s[1], 0.0, h2z);
    if (s == 0) h0[0] = hs[0], h0[1] = hs[1], h20[0] = h2s[0], h20[1] = h2s[1];
  }
  cplx b1[3], b2[3], t[3], t2[3];  // the brackets of E_1 and E_2
  G.forms_z(i, j, hz[0], h0[0], h0[1], vb, 0.0, 0.0, b1);
  G.forms_z(i, j, h2z, h20[0], h20[1], vb, 0.0, 0.0, b2);
  G.forms_z(i, j, hz[0], h0[0], h0[1], xb, 0.0, 0.0, t);
  for (int k = 0; k < 3; ++k) b2[k] += t[k];
  G.forms_z(i, j, hz[1], h0[0], h0[1], vb, 1.0, 0.0, t);  // D_1(w_hat, v)
  G.forms_z(i, j, hz[2], h0[0], h0[1], vb, -1.0, 0.0, t2);
  for (int k = 0; k < 3; ++k) b2[k] += 0.5 * (t[k] - t2[k]);
  if (hp) {
    G.forms_z(i, j, hz[0], h0[0], h0[1], vb, 0.0, 1.0, t);
    G.forms_z(i, j, hz[0], h0[0], h0[1], vb, 0.0, -1.0, t2);
    for (int k = 0; k < 3; ++k) b2[k] += 0.5 * (t[k] - t2[k]);
  }
  // then the w stencil is kept for the forms of w
  cplx W[7][2], d0[3];
#pragma unroll
  for (int s = 0; s < 7; ++s) G.ww(i + di[s], j + dj[s], W[s], un);
  G.forms(i, j, W, vb, 0.0, 0.0, d0);
  G.forms(i, j, W, xb, 0.0, 0.0, t);
  for (int k = 0; k < 3; ++k) b1[k] += t[k];
  G.forms(i, j, W, x2b, 0.0, 0.0, t);
  for (int k = 0; k < 3; ++k) b2[k] += t[k] - d0[k];  // - D(w, v) of D_cc[c', c']
#pragma unroll 1
  for (int s = 0; s < (hp ? 4 : 2); ++s) {  // D_1(w, v), D_1(w, x) and D_cc[c', c'](w, v): +-c', then +-p'
    const double st = (s & 1) ? -1.0 : 1.0, sc = s < 2 ? st : 0.0, sp = s < 2 ? 0.0 : st;
    G.forms(i, j, W, vb, sc, sp, t);
    G.forms(i, j, W, xb, sc, sp, t2);
    for (int k = 0; k < 3; ++k) {
      b1[k] += (0.5 * st) * t[k];
      b2[k] += (0.5 * st) * t2[k];
      if (s < 2) b2[k] += 0.5 * t[k];
    }
  }
#pragma unroll 1
  for (int s = 0; s < (hp ? 4 : 2); ++s) {  // D_c[c''/2](w, v), then D_p[p''/2](w, v)
    const double st = (s & 1) ? -0.5 : 0.5;
    G2.forms(i, j, W, vb, s < 2 ? st : 0.0, s < 2 ? 0.0 : st, t);
    for (int k = 0; k < 3; ++k) b2[k] += st * t[k];
  }
#pragma unroll 1
  for (int s = 0; s < (hp ? 4 : 0); ++s) {  // D_cp[c', p'](w, v)
    const double sc = (s & 2) ? -1.0 : 1.0, sp = (s & 1) ? -1.0 : 1.0;
    G.forms(i, j, W, vb, sc, sp, t);
    for (int k = 0; k < 3; ++k) b2[k] += (0.25 * sc * sp) * t[k];
  }
  const size_t g = (size_t)i * ny + j;
  const cplx iz = to_cplx(ldg(G.fb + 2 * N + g));
  const double je = d.jz_e ? d.jz_e[(size_t)b * d.jz_len + (d.jz_axis == 0 ? i : j)] : 1.0;
  const cplx chi[3] = {mk(1.0 / je, 0.0), mk(1.0 / je, 0.0), -(iz * iz) * je};
  const cplx iz1 = hp ? ldg(a.p1 + o3 + 2 * N + g) : mk(0.0, 0.0), iz2 = hp ? 0.5 * ldg(a.p2 + o3 + 2 * N + g) : mk(0.0, 0.0);
  const cplx chi1 = -2.0 * je * (iz * iz1), chi2 = -je * (2.0 * (iz * iz2) + iz1 * iz1);
  const double pec = 0.9 * 1e8;  // PEC-valued input, as eps_grad
  const bool is_pec[3] = {abs2(to_cplx(ldg(G.fb + g))) >= pec * pec, abs2(to_cplx(ldg(G.fb + N + g))) >= pec * pec, abs2(iz) * pec * pec <= 1.0};
  if constexpr (PERT) {
    cplx f[3][3];
    for (int k = 0; k < 3; ++k) {
      f[0][k] = chi[k] * d0[k];
      f[1][k] = chi[k] * b1[k];
      f[2][k] = chi[k] * b2[k];
      if (k == 2) {
        f[1][k] += chi1 * d0[k];
        f[2][k] += chi1 * b1[k] + chi2 * d0[k];
      }
      if (is_pec[k]) f[0][k] = f[1][k] = f[2][k] = mk(0.0, 0.0);
    }
    pert_site_sums<3>(p, b, g, N, live, f);
  } else {
    const cplx be0 = beta[3 * b], be1 = beta[3 * b + 1], be2 = beta[3 * b + 2];
    cplx *o = map + (size_t)b * 3 * N * M;
    for (int k = 0; k < 3; ++k) {
      cplx e0 = chi[k] * d0[k], e1 = chi[k] * b1[k], e2 = chi[k] * b2[k];
      if (k == 2) {
        e1 += chi1 * d0[k];
        e2 += chi1 * b1[k] + chi2 * d0[k];
      }
      if (is_pec[k]) e0 = e1 = e2 = mk(0.0, 0.0);
      o[((size_t)k * N + g) * M + a.q] = be0 * e0 + be1 * e1 + be2 * e2;
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Tensorial problems: first-order derivatives of the eigenvalue n of mat = msign (-i) M (oracle/tensor_derivatives.py is the
// float64 model) from the sorted right Ritz vectors u and the left ones w of the transposed Krylov-Schur pass, paired mode by
// mode (api.cu).  dn = msign (-i) w^T (dM) u / w^T u.  M has degree <= 2 in the 1-D coefficients, so f dM/df u is exactly
// [M(c + c') - M(c - c')] u / 2; M is affine in the per-site derived fields q of eps' (ft_[0..8]), and the nine
// sensitivities w^T (dM/dq_j) u at a site are the 16 block terms of _eps_terms, which collapse to products of the dual
// intermediate Ub = Dxf^T w1 + Dyf^T w2 (of w), K = Dxb u4 - Dyb u3 (of u) and the site values:
//   (q0, q1, q2) <- (-Ub u1, -Ub u2, Ub K),  q3 <- w3 K,  q4 <- -w4 K,  (S_xx, S_xy) <- (-w4 u1, -w4 u2),  (S_yx, S_yy) <- (w3 u1, w3 u2).
// They are chained through dq/dt' written in q alone (1/t_zz = q2, t_zx/t_zz = q0, t_zy/t_zz = q1, t_yz/t_zz = q3,
// t_xz/t_zz = q4), the PEC model (entries of eps' that are PEC-valued, as tensor_fields_kernel finds them: 0) and the
// congruence eps' = J eps J^T / det J back to the caller's eps_cross: g = J^T g' J / det J.
// ------------------------------------------------------------------------------------------------
template <typename C>
struct TensorDerivArgs {
  int nx, ny, num_modes;
  const cplx *u, *w;             // sorted right Ritz vectors and the paired left ones: slot q of problem b at q vstride + b 4N
  size_t vstride;
  const C *ft;                   // [fb][18][N] derived coefficient fields
  size_t ft_bstride;
  const cplx *cx, *cy;           // [B][4][n] 1-D coefficients
  const cplx *cxp, *cyp, *cxm, *cym;  // [B][4][n] c + f dc/df and c - f dc/df
  const MediumRef *med;          // raw media (PEC marker, congruence), problem b at med[b * med_bstride]
  int med_bstride;
  const cplx *deps;              // [B][9][N] d eps_cross / df (1/Hz) in the eps_cross component order, or null
  double msign;
  cplx *partial;                 // [B*M][nchunk][3]
  const cplx *scale;             // [B][M]: map = gradient numerator * scale
  cplx *map;                     // [B][9][N][M]
};

template <typename C>
__device__ __forceinline__ TensorCell<C> tensor_deriv_cell(const TensorDerivArgs<C> &a, const cplx *vec, int b, int m, const cplx *cx, const cplx *cy) {
  const size_t N = (size_t)a.nx * a.ny;
  const cplx *v = vec + (size_t)m * a.vstride + (size_t)b * 4 * N;
  return TensorCell<C>{v, v + N, v + 2 * N, v + 3 * N, a.ft + a.ft_bstride * b, cx + (size_t)b * 4 * a.nx, cy + (size_t)b * 4 * a.ny, a.nx, a.ny, N};
}

// w^T (d mat / d eps_cross[k](i, j)) u, k in the eps_cross order (not yet divided by w^T u)
template <typename C>
__device__ __forceinline__ void tensor_eps_grad(const TensorDerivArgs<C> &a, const TensorCell<C> &tu, const TensorCell<C> &tw, int b, int i, int j,
                                                cplx g[9]) {
  const size_t s = (size_t)i * a.ny + j;
  const cplx mi = mk(0.0, -a.msign);
  const cplx ub = mi * tw.Ub(i, j), kk = tu.K(i, j);
  const cplx u1 = ldg(tu.ex + s), u2 = ldg(tu.ey + s), w3 = mi * ldg(tw.hx + s), w4 = mi * ldg(tw.hy + s);
  const cplx q0 = to_cplx(tu.F(0, i, j)), q1 = to_cplx(tu.F(1, i, j)), q2 = to_cplx(tu.F(2, i, j));
  const cplx q3 = to_cplx(tu.F(3, i, j)), q4 = to_cplx(tu.F(4, i, j));
  cplx gt[9];  // d/d eps'_ab, row-major
  for (int k = 0; k < 9; ++k) gt[k] = mk(0.0, 0.0);
  const cplx c0 = -(ub * u1), c1 = -(ub * u2), c2 = ub * kk, c3 = w3 * kk, c4 = -(w4 * kk);
  gt[6] = c0 * q2;
  gt[7] = c1 * q2;
  gt[5] = c3 * q2;
  gt[2] = c4 * q2;
  gt[8] = -(q2 * (c0 * q0 + c1 * q1 + c2 * q2 + c3 * q3 + c4 * q4));
  const cplx cs[4] = {-(w4 * u1), -(w4 * u2), w3 * u1, w3 * u2};  // S_xx, S_xy, S_yx, S_yy
  const cplx qa[2] = {q4, q3}, qz[2] = {q0, q1};                 // t_az / t_zz, t_zb / t_zz
  for (int r = 0; r < 2; ++r)
    for (int c = 0; c < 2; ++c) {
      const cplx v = cs[2 * r + c];
      gt[3 * r + c] += v;
      gt[3 * r + 2] -= v * qz[c];
      gt[6 + c] -= v * qa[r];
      gt[8] += v * (qa[r] * qz[c]);
    }
  // the raw congruence at this cell, as tensor_fields_kernel forms it before the PEC model
  const MediumRef &r = a.med[(size_t)b * a.med_bstride];
  const double de = r.p.norm_axis >= 0 ? r.p.de[r.p.norm_axis == 0 ? i : j] : 1.0;
  cplx et[9], mt[9];
  cell_tensors(r.eps, nullptr, (size_t)a.nx * a.ny, s, r.p.a, r.p.b, de, 1.0, et, mt);
  for (int k = 0; k < 9; ++k)
    if (is_pec_val(et[k])) gt[k] = mk(0.0, 0.0);
  const double J[3][3] = {{1, 0, r.p.a}, {0, 1, r.p.b}, {0, 0, de}};
  for (int c = 0; c < 3; ++c)
    for (int d = 0; d < 3; ++d) {
      cplx acc = mk(0.0, 0.0);
      for (int p = 0; p < 3; ++p)
        for (int q = 0; q < 3; ++q)
          if (J[p][c] != 0.0 && J[q][d] != 0.0) acc += (J[p][c] * J[q][d]) * gt[3 * p + q];
      g[3 * c + d] = cdivd(acc, de);
    }
}

// grid (nchunk, B*M), 256 threads: partial sums of w^T u, w^T [M(c + c') - M(c - c')] u / 2 and the material term per chunk
template <typename C>
__global__ void __launch_bounds__(256) tensor_deriv_scan_kernel(TensorDerivArgs<C> a) {
  const int M = a.num_modes, bm = blockIdx.y, b = bm / M, m = bm % M;
  const int ny = a.ny;
  const size_t N = (size_t)a.nx * ny;
  const TensorCell<C> tu = tensor_deriv_cell(a, a.u, b, m, a.cx, a.cy), tw = tensor_deriv_cell(a, a.w, b, m, a.cx, a.cy);
  const TensorCell<C> tp = tensor_deriv_cell(a, a.u, b, m, a.cxp, a.cyp), tm = tensor_deriv_cell(a, a.u, b, m, a.cxm, a.cym);
  const cplx *de = a.deps ? a.deps + (size_t)b * 9 * N : nullptr;
  cplx s_wu = mk(0.0, 0.0), s_da = mk(0.0, 0.0), s_mat = mk(0.0, 0.0);
  for (size_t g = (size_t)blockIdx.x * 256 + threadIdx.x; g < N; g += (size_t)gridDim.x * 256) {
    const int i = (int)(g / ny), j = (int)(g % ny);
    const cplx u0 = ldg(tu.ex + g), u1 = ldg(tu.ey + g), u2 = ldg(tu.hx + g), u3 = ldg(tu.hy + g);
    const cplx w0 = ldg(tw.ex + g), w1 = ldg(tw.ey + g), w2 = ldg(tw.hx + g), w3 = ldg(tw.hy + g);
    s_wu += w0 * u0 + w1 * u1 + w2 * u2 + w3 * u3;
    cplx p[4], q[4];
    tp.apply(i, j, u0, u1, u2, u3, p[0], p[1], p[2], p[3]);
    tm.apply(i, j, u0, u1, u2, u3, q[0], q[1], q[2], q[3]);
    s_da += 0.5 * (w0 * (p[0] - q[0]) + w1 * (p[1] - q[1]) + w2 * (p[2] - q[2]) + w3 * (p[3] - q[3]));
    if (de) {
      cplx gr[9];
      tensor_eps_grad(a, tu, tw, b, i, j, gr);
      for (int k = 0; k < 9; ++k) s_mat += gr[k] * ldg(de + (size_t)k * N + g);
    }
  }
  __shared__ cplx red[3][256];
  red[0][threadIdx.x] = s_wu;
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

// grid (nchunk, B*M), 256 threads: per chunk, sum_g sum_c (w^T d mat / d eps_cross[c](g) u) delta eps_k,c(g) for k < p.npert
// (p: nine components per perturbation), partials laid out as deriv_pert_kernel's
template <typename C>
__global__ void __launch_bounds__(256) tensor_pert_kernel(TensorDerivArgs<C> a, PertArgs p) {
  const int M = a.num_modes, bm = blockIdx.y, b = bm / M, m = bm % M;
  const int ny = a.ny;
  const size_t N = (size_t)a.nx * ny;
  const TensorCell<C> tu = tensor_deriv_cell(a, a.u, b, m, a.cx, a.cy), tw = tensor_deriv_cell(a, a.w, b, m, a.cx, a.cy);
  const cplx *pe = p.eps + p.bstride * b;
  cplx s[kPertGroup];
#pragma unroll
  for (int k = 0; k < kPertGroup; ++k) s[k] = mk(0.0, 0.0);
  for (size_t g = (size_t)blockIdx.x * 256 + threadIdx.x; g < N; g += (size_t)gridDim.x * 256) {
    const int i = (int)(g / ny), j = (int)(g % ny);
    cplx gr[9];
    tensor_eps_grad(a, tu, tw, b, i, j, gr);
#pragma unroll
    for (int k = 0; k < kPertGroup; ++k)
      if (k < p.npert) {
        const cplx *e = pe + k * p.kstride + g;
        cplx acc = mk(0.0, 0.0);
        for (int c = 0; c < 9; ++c) acc += gr[c] * ldg(e + (size_t)c * N);
        s[k] += acc;
      }
  }
  __shared__ cplx red[kPertGroup][256];
  for (int k = 0; k < kPertGroup; ++k) red[k][threadIdx.x] = s[k];
  __syncthreads();
  for (int h = 128; h > 0; h >>= 1) {
    if ((int)threadIdx.x < h)
      for (int k = 0; k < kPertGroup; ++k) red[k][threadIdx.x] += red[k][threadIdx.x + h];
    __syncthreads();
  }
  if (threadIdx.x < kPertGroup)
    p.partial[(((size_t)bm * (kPertGroup / 3) + threadIdx.x / 3) * gridDim.x + blockIdx.x) * 3 + threadIdx.x % 3] = red[threadIdx.x][0];
}

// grid like epilogue_kernel: map[b][k][g][m] = (w^T d mat / d eps_cross[k](g) u) * scale[b][m]
template <typename C>
__global__ void __launch_bounds__(256) tensor_deriv_map_kernel(TensorDerivArgs<C> a) {
  const int nx = a.nx, ny = a.ny, M = a.num_modes;
  const size_t N = (size_t)nx * ny;
  const int j = blockIdx.x * 64 + threadIdx.x, i = blockIdx.y * 4 + threadIdx.y;
  const int m = blockIdx.z % M, b = blockIdx.z / M;
  if (i >= nx || j >= ny) return;
  const TensorCell<C> tu = tensor_deriv_cell(a, a.u, b, m, a.cx, a.cy), tw = tensor_deriv_cell(a, a.w, b, m, a.cx, a.cy);
  cplx gr[9];
  tensor_eps_grad(a, tu, tw, b, i, j, gr);
  const cplx sc = a.scale[(size_t)b * M + m];
  const size_t g = (size_t)i * ny + j;
  cplx *o = a.map + (size_t)b * 9 * N * M;
  for (int k = 0; k < 9; ++k) o[((size_t)k * N + g) * M + m] = gr[k] * sc;
}

}  // namespace b200ms
