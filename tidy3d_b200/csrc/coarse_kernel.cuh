// Fused multigrid tail: the V-cycle on all levels from `l0` down to the coarsest one in ONE kernel, one CTA per problem,
// with the level vectors held in shared memory.  On those levels (<= 32^2 .. 64^2 cells) the separate kernels of the
// unfused cycle are pure launch / dependency latency: ~45 short launches per V-cycle whatever the batch size; fused they are a few dozen block-synchronised passes over a few thousand cells.
// The arithmetic is that of BatchSolver::vcycle (jacobi0, nu-1 pre-sweeps, residual, restriction, recursion, prolongation,
// nu post-sweeps; n_sw Jacobi sweeps on the coarsest level) with the stored omega/diag smoother.
#pragma once
#include "kernels.cuh"

namespace b200ms {

constexpr int kFusedMaxLevels = 6;

template <typename P, typename PC>
struct FusedLevel {
  int nx, ny;
  const PC *fields;      // [fB][nf][N]
  size_t fbstride;
  const P *cx, *cy;      // [B][4][n]
  const P *dinv;         // [B][2][N]
  TransferArgs tr;       // to the next coarser level (unused on the last one)
};
template <typename P, typename PC>
struct FusedArgs {
  int nl, nu, ncoarse;   // levels, pre/post sweeps, sweeps on the coarsest level (incl. the first one from zero)
  FusedLevel<P, PC> lv[kFusedMaxLevels];
  const P *rin;          // [B][2][N0] right-hand side on level l0
  P *xout;               // [B][2][N0] result
  const P *sigma;        // [B]
};

// shared-memory footprint in elements of P: per level x, b, tmp (2N each) + u, t (N each)
inline size_t fused_smem_elems(const int *nxs, const int *nys, int nl) {
  size_t e = 0;
  for (int l = 0; l < nl; ++l) e += (size_t)8 * nxs[l] * nys[l];
  return e;
}

template <typename P, typename PC, bool HAS_MU>
struct FusedOps {
  // u, t of the whole level from x (zero outside the grid)
  static __device__ void ut(const FusedLevel<P, PC> &L, int b, const P *x, P *u, P *t) {
    const int nx = L.nx, ny = L.ny;
    const size_t N = (size_t)nx * ny;
    const PC *fb = L.fields + L.fbstride * b;
    const PC *exx = fb, *eyy = fb + N, *iez = fb + 2 * N, *imz = fb + 5 * N;
    const P *cx = L.cx + (size_t)b * 4 * nx, *cy = L.cy + (size_t)b * 4 * ny;
    const P *v1 = x, *v2 = x + N;
    const P z = zero_of<P>();
    for (int c = threadIdx.x; c < (int)N; c += blockDim.x) {
      const int i = c / ny, j = c % ny;
      const P a00 = ldg(exx + c) * v1[c], b00 = ldg(eyy + c) * v2[c];
      const P am = i > 0 ? ldg(exx + c - ny) * v1[c - ny] : z;
      const P bm = j > 0 ? ldg(eyy + c - 1) * v2[c - 1] : z;
      u[c] = -(ldg(iez + c) * (ldg(cx + 2 * nx + i) * a00 + ldg(cx + 3 * nx + i) * am + ldg(cy + 2 * ny + j) * b00 + ldg(cy + 3 * ny + j) * bm));
      const P v2n = i + 1 < nx ? v2[c + ny] : z, v1n = j + 1 < ny ? v1[c + 1] : z;
      P tt = ldg(cx + i) * v2[c] + ldg(cx + nx + i) * v2n - ldg(cy + j) * v1[c] - ldg(cy + ny + j) * v1n;
      if (HAS_MU) tt = ldg(imz + c) * tt;
      t[c] = tt;
    }
  }
  // mode 0: y = dinv * rhs;  mode 1: y = x + dinv * (rhs - (A - sigma) x);  mode 2: y = rhs - (A - sigma) x.   u, t from ut(x)
  static __device__ void sweep(const FusedLevel<P, PC> &L, int b, int mode, const P *x, const P *rhs, const P *u, const P *t, P sg, P *y) {
    const int nx = L.nx, ny = L.ny;
    const size_t N = (size_t)nx * ny;
    const P *dinv = L.dinv + (size_t)b * 2 * N;
    if (mode == 0) {
      for (int e = threadIdx.x; e < (int)(2 * N); e += blockDim.x) y[e] = ldg(dinv + e) * rhs[e];
      return;
    }
    const PC *fb = L.fields + L.fbstride * b;
    const PC *exx = fb, *eyy = fb + N, *mxx = fb + 3 * N, *myy = fb + 4 * N;
    const P *cx = L.cx + (size_t)b * 4 * nx, *cy = L.cy + (size_t)b * 4 * ny;
    const P z = zero_of<P>();
    for (int c = threadIdx.x; c < (int)N; c += blockDim.x) {
      const int i = c / ny, j = c % ny;
      const P u00 = u[c], u10 = i + 1 < nx ? u[c + ny] : z, u01 = j + 1 < ny ? u[c + 1] : z;
      const P t00 = t[c], tm0 = i > 0 ? t[c - ny] : z, t0m = j > 0 ? t[c - 1] : z;
      const P v1 = x[c], v2 = x[N + c];
      const P pa = ldg(exx + c) * v1, pb = ldg(eyy + c) * v2;
      P p1 = ldg(cx + i) * u00 + ldg(cx + nx + i) * u10;
      P p2 = ldg(cy + j) * u00 + ldg(cy + ny + j) * u01;
      const P c1 = ldg(cy + 2 * ny + j) * t00 + ldg(cy + 3 * ny + j) * t0m - pa;
      const P c2 = ldg(cx + 2 * nx + i) * t00 + ldg(cx + 3 * nx + i) * tm0 + pb;
      if (HAS_MU) { p1 += ldg(myy + c) * c1; p2 -= ldg(mxx + c) * c2; } else { p1 += c1; p2 -= c2; }
      const P o1 = p1 - sg * v1, o2 = p2 - sg * v2;
      if (mode == 2) {
        y[c] = rhs[c] - o1;
        y[N + c] = rhs[N + c] - o2;
      } else {
        y[c] = v1 + ldg(dinv + c) * (rhs[c] - o1);
        y[N + c] = v2 + ldg(dinv + N + c) * (rhs[N + c] - o2);
      }
    }
  }
  static __device__ void restrict_to(const TransferArgs &a, const P *fine, P *coarse) {
    const size_t Nf = (size_t)a.nxf * a.nyf, Nc = (size_t)a.nxc * a.nyc;
    for (int e = threadIdx.x; e < (int)(2 * Nc); e += blockDim.x) {
      const int comp = e >= (int)Nc, cc = e - comp * (int)Nc, I = cc / a.nyc, J = cc % a.nyc;
      const Transfer1DDev &tx = comp == 0 ? a.xe : a.xn;
      const Transfer1DDev &ty = comp == 0 ? a.yn : a.ye;
      const P *f = fine + (size_t)comp * Nf;
      P acc = zero_of<P>();
      for (int kx = tx.r_ptr[I]; kx < tx.r_ptr[I + 1]; ++kx) {
        const P *row = f + (size_t)tx.r_idx[kx] * a.nyf;
        P racc = zero_of<P>();
        for (int ky = ty.r_ptr[J]; ky < ty.r_ptr[J + 1]; ++ky) racc += (typename RealOf<P>::type)ty.r_w[ky] * row[ty.r_idx[ky]];
        acc += (typename RealOf<P>::type)tx.r_w[kx] * racc;
      }
      if ((comp == 0 && a.mask_y && J == 0 && a.nyc > 1) || (comp == 1 && a.mask_x && I == 0 && a.nxc > 1)) acc = zero_of<P>();
      coarse[e] = acc;
    }
  }
  static __device__ void prolong_add(const TransferArgs &a, const P *coarse, P *fine) {
    const size_t Nf = (size_t)a.nxf * a.nyf, Nc = (size_t)a.nxc * a.nyc;
    for (int e = threadIdx.x; e < (int)(2 * Nf); e += blockDim.x) {
      const int comp = e >= (int)Nf, cc = e - comp * (int)Nf, i = cc / a.nyf, j = cc % a.nyf;
      if ((comp == 0 && a.mask_y && j == 0 && a.nyf > 1) || (comp == 1 && a.mask_x && i == 0 && a.nxf > 1)) continue;
      const Transfer1DDev &tx = comp == 0 ? a.xe : a.xn;
      const Transfer1DDev &ty = comp == 0 ? a.yn : a.ye;
      const P *c = coarse + (size_t)comp * Nc;
      const int I0 = tx.p_i0[i], I1 = tx.p_i1[i], J0 = ty.p_i0[j], J1 = ty.p_i1[j];
      using R = typename RealOf<P>::type;
      const R wx0 = (R)tx.p_w0[i], wx1 = (R)tx.p_w1[i], wy0 = (R)ty.p_w0[j], wy1 = (R)ty.p_w1[j];
      fine[e] = fine[e] + (wx0 * (wy0 * c[(size_t)I0 * a.nyc + J0] + wy1 * c[(size_t)I0 * a.nyc + J1]) +
                           wx1 * (wy0 * c[(size_t)I1 * a.nyc + J0] + wy1 * c[(size_t)I1 * a.nyc + J1]));
    }
  }
};

template <typename P, typename PC, bool HAS_MU>
__global__ void __launch_bounds__(512) fused_vcycle_kernel(FusedArgs<P, PC> a) {
  extern __shared__ __align__(16) unsigned char fused_smem[];
  using Ops = FusedOps<P, PC, HAS_MU>;
  const int b = blockIdx.x;
  P *base = reinterpret_cast<P *>(fused_smem);
  P *X[kFusedMaxLevels], *Bv[kFusedMaxLevels], *Tm[kFusedMaxLevels], *U[kFusedMaxLevels], *Tt[kFusedMaxLevels];
  {
    size_t off = 0;
    for (int l = 0; l < a.nl; ++l) {
      const size_t N = (size_t)a.lv[l].nx * a.lv[l].ny;
      X[l] = base + off; Bv[l] = X[l] + 2 * N; Tm[l] = Bv[l] + 2 * N; U[l] = Tm[l] + 2 * N; Tt[l] = U[l] + N;
      off += 8 * N;
    }
  }
  const P sg = ldg(a.sigma + b);
  {
    const size_t N0 = (size_t)a.lv[0].nx * a.lv[0].ny;
    const P *r = a.rin + (size_t)b * 2 * N0;
    for (int e = threadIdx.x; e < (int)(2 * N0); e += blockDim.x) Bv[0][e] = r[e];
  }
  __syncthreads();
  auto smooth = [&](int l, int nsweeps, bool from_zero) {  // result in X[l]
    for (int s = 0; s < nsweeps; ++s) {
      if (s == 0 && from_zero) {
        Ops::sweep(a.lv[l], b, 0, nullptr, Bv[l], nullptr, nullptr, sg, X[l]);
        __syncthreads();
        continue;
      }
      Ops::ut(a.lv[l], b, X[l], U[l], Tt[l]);
      __syncthreads();
      Ops::sweep(a.lv[l], b, 1, X[l], Bv[l], U[l], Tt[l], sg, Tm[l]);
      __syncthreads();
      P *sw = X[l]; X[l] = Tm[l]; Tm[l] = sw;
    }
  };
  for (int l = 0; l + 1 < a.nl; ++l) {  // down
    smooth(l, a.nu, true);
    Ops::ut(a.lv[l], b, X[l], U[l], Tt[l]);
    __syncthreads();
    Ops::sweep(a.lv[l], b, 2, X[l], Bv[l], U[l], Tt[l], sg, Tm[l]);
    __syncthreads();
    Ops::restrict_to(a.lv[l].tr, Tm[l], Bv[l + 1]);
    __syncthreads();
  }
  smooth(a.nl - 1, a.ncoarse, true);
  for (int l = a.nl - 2; l >= 0; --l) {  // up
    Ops::prolong_add(a.lv[l].tr, X[l + 1], X[l]);
    __syncthreads();
    smooth(l, a.nu, false);
  }
  {
    const size_t N0 = (size_t)a.lv[0].nx * a.lv[0].ny;
    P *o = a.xout + (size_t)b * 2 * N0;
    for (int e = threadIdx.x; e < (int)(2 * N0); e += blockDim.x) o[e] = X[0][e];
  }
}

}  // namespace b200ms
