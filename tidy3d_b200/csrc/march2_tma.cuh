// Pair-marching stencil with TMA row staging (cp.async.bulk + mbarrier), sm_90a.
//
// Same march and the same arithmetic as stencil_march2_kernel (csrc/march2.cuh); what changes is how a row reaches the thread
// that owns it.  A strip's slice of a grid row is contiguous in HBM (W column pairs = 8 W bytes per array), so one elected
// thread moves it with a bulk asynchronous copy -- one `cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes` per
// array and row: v1, v2, exx, eyy, 1/ezz of row k+2 and rhs / omega-over-diagonal of row k -- into a ring of D stages in shared
// memory, and every stage completes on its own mbarrier (expect_tx = the bytes of that step).  Rows in flight cost no registers
// and no per-thread load instructions: with D = 3 two to three rows (18 KB each at W = 256) are in flight per CTA, against one
// row of prefetch registers in the register version, which is what the register version's bandwidth is limited by
// (Little's law: bytes in flight per SM = HBM bandwidth x latency / SMs).  A stage is refilled by the elected thread right after the
// __syncthreads that ends the step which consumed it (the march needs that barrier anyway), so no "empty" barriers exist.
// Requirements beyond the register version: ny % 4 == 0 (16-byte aligned row slices).  MODE_JACOBI_D0 stays with the register
// version.  A wait that does not complete within ~2^24 polls traps instead of hanging the device.
//
// MODE_RESID_RESTRICT: the residual followed by the restriction to the next coarser level, without storing the fine residual.
// A CTA owns the coarse rows [I0, I0 + rows) (rows = coarse rows here) and marches the fine rows their restriction lists
// reach (Ex: x-edge lists, Ey: x-node lists); the fine rows two neighbouring CTAs both need are computed by both.  Each
// residual row goes to a ring of kRrRing rows in shared memory, and a coarse row is formed as soon as the last fine row
// of its lists is there, by restrict4_kernel's expression in restrict4_kernel's order (csrc/kernels.cuh).  One strip per
// row (ny <= 2 kM2MaxW), packed lists on all four axes; the host checks that no coarse row needs a fine row older than the
// ring holds (resid_restrict_plan in csrc/solver.cuh).
#pragma once

namespace b200ms {

__device__ __forceinline__ unsigned smem_u32(const void *p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long *bar, unsigned count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(unsigned long long *bar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(unsigned long long *bar, unsigned parity) {
  unsigned ok;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
      "selp.u32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(unsigned long long *bar, unsigned parity) {
  unsigned spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++spins > (1u << 24)) __trap();
  }
}
__device__ __forceinline__ void bulk_g2s(void *smem_dst, const void *gmem_src, unsigned bytes, unsigned long long *bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];\n" ::"r"(smem_u32(smem_dst)), "l"(gmem_src),
               "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
// one 4-byte asynchronous copy (LDGSTS), and an arrival on `bar` once this thread's earlier ones have landed (the barrier's
// expected arrival count includes it)
__device__ __forceinline__ void cp_async4(void *smem_dst, const void *gmem_src) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;\n" ::"r"(smem_u32(smem_dst)), "l"(gmem_src) : "memory");
}
__device__ __forceinline__ void cp_async_arrive(unsigned long long *bar) {
  asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];\n" ::"r"(smem_u32(bar)) : "memory");
}

template <int MODE>
struct M2TmaArrays {
  static constexpr int n = 5 + (MODE != MODE_APPLY ? 2 : 0) + (MODE == MODE_JACOBI_D ? 2 : 0);
};

constexpr int kRrRing = 8;  // residual rows held for the restriction (power of two)

// dynamic shared memory of MODE_RESID_RESTRICT beyond the row ring: residual ring [kRrRing][2][ny] floats, then the fine-row
// range of the CTA and the last fine row of each of its coarse rows
inline size_t rr_smem_extra(int ny) { return (size_t)kRrRing * 2 * ny * sizeof(float) + (2 + kM2MaxSteps) * sizeof(int); }

template <int MODE, int D>
__global__ void __launch_bounds__(kM2MaxW, 2) stencil_march2_tma_kernel(StencilArgs<float, float> a, int rows) {
  static_assert(MODE == MODE_APPLY || MODE == MODE_RESID || MODE == MODE_JACOBI_D || MODE == MODE_RESID_RESTRICT,
                "TMA pair kernel: apply / residual / stored-diagonal sweep / residual + restriction");
  static_assert(kM2Unroll % D == 0, "ring depth must divide the unroll factor");
  using T = float;
  using V = float2;
  constexpr bool HAS_RHS = (MODE != MODE_APPLY);
  constexpr bool DSTORED = (MODE == MODE_JACOBI_D);
  constexpr bool RESTR = (MODE == MODE_RESID_RESTRICT);
  constexpr int NARR = M2TmaArrays<MODE>::n;
  __shared__ T sB[2][kM2MaxW + 2], sV[2][kM2MaxW + 2], sU[2][kM2MaxW + 2], sTt[2][kM2MaxW + 2];
  __shared__ RowCoef<T> sX[kM2MaxSteps + 2];
  __shared__ __align__(8) unsigned long long sBar[D];
  extern __shared__ __align__(128) unsigned char m2_ring_raw[];  // [D][NARR][W] float2
  V *ring = reinterpret_cast<V *>(m2_ring_raw);

  const int nx = a.nx, ny = a.ny;
  const int W = blockDim.x;
  const unsigned N = (unsigned)nx * (unsigned)ny;
  const int b = blockIdx.z;
  const int c = threadIdx.x;
  const int npairs = ny >> 1;
  const int q0 = (int)blockIdx.x * (W - 2);  // first column pair of the strip
  const int q = q0 + c;
  const int gj = 2 * q;
  int i0 = blockIdx.y * rows;
  int iend = (i0 + rows < nx) ? i0 + rows : nx;
  int k0 = i0 - 3;
  int nsteps = rows + 3;
  const bool colv = q < npairs;
  const bool outc = colv && (c >= 1 || blockIdx.x == 0) && (c <= W - 2 || q == npairs - 1);
  // MODE_RESID_RESTRICT: the CTA's coarse rows [I0, I1) and the fine rows [i0, iend) their restriction lists reach
  T *sRes = nullptr;
  int *sRng = nullptr;
  int I0 = 0, I1 = 0;
  if constexpr (RESTR) {
    sRes = reinterpret_cast<T *>(m2_ring_raw + (size_t)D * NARR * W * sizeof(V));
    sRng = reinterpret_cast<int *>(sRes + (size_t)kRrRing * 2 * ny);
    I0 = blockIdx.y * rows;
    I1 = min(I0 + rows, a.tr->nxc);
    if (c == 0) { sRng[0] = nx; sRng[1] = -1; }
    __syncthreads();
    if (c < I1 - I0) {
      const int4 xe = __ldg(reinterpret_cast<const int4 *>(a.tr->xe.r4 + I0 + c)), xn = __ldg(reinterpret_cast<const int4 *>(a.tr->xn.r4 + I0 + c));
      const int hi = max(xe.w, xn.w);  // packed lists ascend and repeat their last index
      sRng[2 + c] = hi;
      atomicMin(&sRng[0], min(xe.x, xn.x));
      atomicMax(&sRng[1], hi);
    }
    __syncthreads();
    i0 = sRng[0];
    iend = sRng[1] + 1;
    nsteps = kM2Unroll * ((iend - i0 + 3 + kM2Unroll - 1) / kM2Unroll);
    k0 = i0 - 3;
  }
  const T *x1 = a.x + (size_t)b * 2 * N, *x2 = x1 + N;
  const T *fb = a.fields + a.field_bstride * b;
  const T *exx = fb, *eyy = fb + N, *iez = fb + 2 * (size_t)N;
  const T *cx = a.cx + (size_t)b * 4 * nx, *cy = a.cy + (size_t)b * 4 * ny;
  const T *r1 = HAS_RHS ? a.rhs + (size_t)b * 2 * N : nullptr, *r2 = HAS_RHS ? r1 + N : nullptr;
  const T *d1 = DSTORED ? a.dinv + (size_t)b * 2 * N : nullptr, *d2 = DSTORED ? d1 + N : nullptr;
  T *y1 = a.y + (size_t)b * 2 * N, *y2 = y1 + N;
  const T zT = 0.0f;
  const V zV = {zT, zT};
  const int wcopy = (npairs - q0 < W) ? npairs - q0 : W;  // column pairs of this strip that exist
  const unsigned nbytes = (unsigned)wcopy * (unsigned)sizeof(V);
  const int raw_lo = (i0 - 1 > 0) ? i0 - 1 : 0;
  const int raw_hi = RESTR ? min(iend, nx - 1) : (i0 + rows < nx - 1) ? i0 + rows : nx - 1;

  // lanes 0 .. NARR-1 of warp 0 each own one array: lane 0 arms the stage of step jj (expect_tx = the bytes of that step), then
  // every owner lane issues the bulk copy of its array's row slice
  const T *my_arr = nullptr;
  if (c == 0) my_arr = x1; else if (c == 1) my_arr = x2; else if (c == 2) my_arr = exx; else if (c == 3) my_arr = eyy; else if (c == 4) my_arr = iez;
  else if (c == 5) my_arr = r1; else if (c == 6) my_arr = r2; else if (c == 7) my_arr = d1; else if (c == 8) my_arr = d2;
  my_arr += 2 * (size_t)q0;
  const bool my_raw = c < 5;
  auto issue = [&](int jj, int stage) {
    const int gr = k0 + jj + 2, go = k0 + jj;
    const bool rawv = gr >= raw_lo && gr <= raw_hi;
    const bool outv = HAS_RHS && go >= i0 && go < iend;
    unsigned long long *bar = &sBar[stage];
    if (c == 0) mbar_expect_tx(bar, (rawv ? 5u : 0u) * nbytes + (outv ? (unsigned)(NARR - 5) : 0u) * nbytes);
    const bool mine = my_raw ? rawv : outv;
    if (mine) bulk_g2s(ring + ((size_t)stage * NARR + c) * W, my_arr + (size_t)(my_raw ? gr : go) * ny, nbytes, bar);
  };

  if (c == 0) {
#pragma unroll
    for (int s = 0; s < D; ++s) mbar_init(&sBar[s], 1);
    mbar_fence_init();
  }
  for (int r = c; r < nsteps + 1; r += W) {  // coefficients of rows k0 .. k0 + nsteps
    const int gi = k0 + r;
    RowCoef<T> rc;
    rc.f0 = rc.f1 = rc.b0 = rc.bm = zT;
    if (gi >= 0 && gi < nx) { rc.f0 = __ldg(cx + gi); rc.f1 = __ldg(cx + nx + gi); rc.b0 = __ldg(cx + 2 * nx + gi); rc.bm = __ldg(cx + 3 * nx + gi); }
    sX[r] = rc;
  }
  for (int s = 0; s < 2; ++s) { sB[s][c + 1] = zT; sV[s][c + 1] = zT; sU[s][c + 1] = zT; sTt[s][c + 1] = zT; }
  if (c < 2)
    for (int s = 0; s < 2; ++s) {
      const int e = c == 0 ? 0 : W + 1;
      sB[s][e] = zT; sV[s][e] = zT; sU[s][e] = zT; sTt[s][e] = zT;
    }
  V yf0 = zV, yf1 = zV, yb0 = zV, ybm = zV;
  if (colv) { yf0 = ldg2(cy + gj); yf1 = ldg2(cy + ny + gj); yb0 = ldg2(cy + 2 * ny + gj); ybm = ldg2(cy + 3 * ny + gj); }
  const T sg = __ldg(a.sigma + b);
  __syncthreads();  // barriers initialised, coefficient rows and exchange rows in place
  if (c < NARR) {
#pragma unroll
    for (int s = 0; s < D; ++s)
      if (s < nsteps) issue(s, s);
  }

  // coarse row I of both components out of the residual ring: restrict4_kernel's sums in its order, with its contractions
  int nI = I0;
  auto restrict_row = [&](int I) {
    const TransferArgs &t = *a.tr;
    const int nyc = t.nyc;
    const size_t Nc = (size_t)t.nxc * nyc;
    for (int o = c; o < 2 * nyc; o += W) {
      const int comp = o >= nyc ? 1 : 0, J = o - comp * nyc;
      const RList4 *tx = comp == 0 ? t.xe.r4 : t.xn.r4, *ty = comp == 0 ? t.yn.r4 : t.ye.r4;
      const int4 xi = __ldg(reinterpret_cast<const int4 *>(tx + I)), yi = __ldg(reinterpret_cast<const int4 *>(ty + J));
      const float4 xw = __ldg(reinterpret_cast<const float4 *>(tx + I) + 1), yw = __ldg(reinterpret_cast<const float4 *>(ty + J) + 1);
      const int ix[4] = {xi.x, xi.y, xi.z, xi.w}, iy[4] = {yi.x, yi.y, yi.z, yi.w};
      const float wx[4] = {xw.x, xw.y, xw.z, xw.w}, wy[4] = {yw.x, yw.y, yw.z, yw.w};
      T acc = 0.0f;
#pragma unroll
      for (int p = 0; p < 4; ++p) {
        const T *row = sRes + (size_t)(ix[p] & (kRrRing - 1)) * 2 * ny + comp * ny;
        T racc = 0.0f;
#pragma unroll
        for (int qq = 0; qq < 4; ++qq) racc = __fmaf_rn(wy[qq], row[iy[qq]], racc);
        acc = __fmaf_rn(wx[p], racc, acc);
      }
      if ((comp == 0 && t.mask_y && J == 0 && nyc > 1) || (comp == 1 && t.mask_x && I == 0 && t.nxc > 1)) acc = 0.0f;
      a.coarse[((size_t)b * 2 + comp) * Nc + (size_t)I * nyc + J] = acc;
    }
  };
  (void)restrict_row;

  V a1 = zV, b1 = zV, v11 = zV, v21 = zV, a0 = zV, b0 = zV, v10 = zV, v20 = zV, ie1 = zV;
  V u0 = zV, t0 = zV, tm = zV;
  RowCoef<T> xc = sX[0];  // coefficients of row k

  for (int j0 = 0; j0 < nsteps; j0 += kM2Unroll) {
    const unsigned parity0 = (unsigned)(j0 / D);  // ring pass of the first step of this group (kM2Unroll / D passes per group)
#pragma unroll
    for (int u = 0; u < kM2Unroll; ++u) {
      const int j = j0 + u, k = k0 + j;
      const int s = u & 1, sp = s ^ 1;
      const int stage = u % D;
      const unsigned parity = (parity0 + (unsigned)(u / D)) & 1u;
      const int gr = k + 2;
      const bool rawv = gr >= raw_lo && gr <= raw_hi;
      const bool outv = HAS_RHS && k >= i0 && k < iend;
      // step 0: row k+2 (and rhs / diagonal of row k) out of the ring
      mbar_wait(&sBar[stage], parity);
      const V *st = ring + (size_t)stage * NARR * W;
      V v12 = zV, v22 = zV, ex2 = zV, ey2 = zV, ie2 = zV;
      if (rawv && colv) { v12 = st[0 * W + c]; v22 = st[1 * W + c]; ex2 = st[2 * W + c]; ey2 = st[3 * W + c]; ie2 = st[4 * W + c]; }
      V cr1 = zV, cr2 = zV, cd1 = zV, cd2 = zV;
      if (HAS_RHS && outv && outc) {
        cr1 = st[5 * W + c]; cr2 = st[6 * W + c];
        if (DSTORED) { cd1 = st[7 * W + c]; cd2 = st[8 * W + c]; }
      }
      V a2, b2;
      a2.x = ex2.x * v12.x; a2.y = ex2.y * v12.y;
      b2.x = ey2.x * v22.x; b2.y = ey2.y * v22.y;
      // step 1: publish what the neighbouring pairs need of row k+2
      sB[s][c + 1] = b2.y;
      sV[s][c + 1] = v12.x;
      // step 2: u[k+1], t[k+1]
      const T bl = sB[sp][c], v1r = sV[sp][c + 2];
      const RowCoef<T> xn = sX[j + 1];
      V u1, t1;
      u1.x = -(ie1.x * (xn.b0 * a1.x + xn.bm * a0.x + yb0.x * b1.x + ybm.x * bl));
      u1.y = -(ie1.y * (xn.b0 * a1.y + xn.bm * a0.y + yb0.y * b1.y + ybm.y * b1.x));
      t1.x = xn.f0 * v21.x + xn.f1 * v22.x - yf0.x * v11.x - yf1.x * v11.y;
      t1.y = xn.f0 * v21.y + xn.f1 * v22.y - yf0.y * v11.y - yf1.y * v1r;
      sU[s][c + 1] = u1.x;
      sTt[s][c + 1] = t1.y;
      // step 3: outputs of row k
      if (outc && k >= i0 && k < iend) {
        const T ur = sU[sp][c + 2], tl = sTt[sp][c];
        T p1x = xc.f0 * u0.x + xc.f1 * u1.x, p1y = xc.f0 * u0.y + xc.f1 * u1.y;
        T p2x = yf0.x * u0.x + yf1.x * u0.y, p2y = yf0.y * u0.y + yf1.y * ur;
        const T c1x = yb0.x * t0.x + ybm.x * tl - a0.x, c1y = yb0.y * t0.y + ybm.y * t0.x - a0.y;
        const T c2x = xc.b0 * t0.x + xc.bm * tm.x + b0.x, c2y = xc.b0 * t0.y + xc.bm * tm.y + b0.y;
        p1x += c1x; p1y += c1y; p2x -= c2x; p2y -= c2y;
        const T o1x = p1x - sg * v10.x, o1y = p1y - sg * v10.y, o2x = p2x - sg * v20.x, o2y = p2y - sg * v20.y;
        const unsigned g = (unsigned)k * (unsigned)ny + (unsigned)gj;
        if (MODE == MODE_APPLY) {
          stg2(y1 + g, o1x, o1y); stg2(y2 + g, o2x, o2y);
        } else if (MODE == MODE_RESID) {
          stg2(y1 + g, cr1.x - o1x, cr1.y - o1y); stg2(y2 + g, cr2.x - o2x, cr2.y - o2y);
        } else if (RESTR) {
          T *rr = sRes + (size_t)(k & (kRrRing - 1)) * 2 * ny + gj;
          *reinterpret_cast<V *>(rr) = make_float2(cr1.x - o1x, cr1.y - o1y);
          *reinterpret_cast<V *>(rr + ny) = make_float2(cr2.x - o2x, cr2.y - o2y);
        } else {
          stg2(y1 + g, v10.x + cd1.x * (cr1.x - o1x), v10.y + cd1.y * (cr1.y - o1y));
          stg2(y2 + g, v20.x + cd2.x * (cr2.x - o2x), v20.y + cd2.y * (cr2.y - o2y));
        }
      }
      tm = t0; t0 = t1; u0 = u1;
      a0 = a1; b0 = b1; v10 = v11; v20 = v21; a1 = a2; b1 = b2; v11 = v12; v21 = v22;
      ie1 = ie2;
      xc = xn;
      __syncthreads();
      // every thread has read stage `stage`: refill it with the rows of step j + D
      if (c < NARR && j + D < nsteps) issue(j + D, stage);
      if constexpr (RESTR) {
        // the coarse rows whose last fine row is row k (the ring still holds their first one: resid_restrict_plan)
        while (nI < I1 && k >= sRng[2 + nI - I0]) {
          restrict_row(nI);
          ++nI;
        }
      }
    }
  }
}

// MODE_PROLONG_JACOBI2: the post-smoothing half of a V(2,2) level in one march -- the prolongation x = x_old + P e_c and two
// stored-diagonal sweeps -- in place of prolong_add4_kernel (prolong_add_kernel) and two MODE_JACOBI_D passes.  Row step j
// (row k = k0 + j) runs three stages:
//   0. raw row k+2: x_old out of the ring plus P e_c, prolong_add4_kernel's sum with its contractions; the four coarse rows
//      it reads (x-edge lists for component 0, x-node lists for component 1) are staged into the same ring stage by 4-byte
//      cp.async that arrive on the stage's barrier (coarse rows need not be 16-byte aligned);
//   1. sweep 1 (the march of stencil_march2_tma_kernel<MODE_JACOBI_D>) with output row k, kept in the thread's registers;
//   2. sweep 2, the same march one pipeline later: row k of sweep 1 is its newest row, its output row k - 2 goes to a.y.
// Sweep 2 needs exx / eyy / 1/ezz of row k and rhs / omega-over-diagonal of row k - 2: the ring stage of step j - 2 holds
// both, so the ring has kPjRing = 4 stages (steps j - 2 .. j and one in flight) and a stage is refilled once sweep 2 has
// read it.  A CTA owns the output rows [i0, i0 + rows); it runs sweep 1 on [i0 - 1, i0 + rows] and the prolongation on
// [i0 - 2, i0 + rows + 1], rows its neighbours also compute.  One strip per row; rows % 6 == 0 and rows + 6 <= kM2MaxSteps
// (host: fused_post_plan in csrc/solver.cuh).  a.y never aliases a.x.
// The row-step arithmetic carries explicit roundings (pj_u, pj_t, pj_sweep): the contractions the compiler gives
// stencil_march2_tma_kernel<MODE_JACOBI_D> (its PTX, plus the multiply-subtract pairs ptxas fuses) depend on the code around
// the expressions, so the same source in this kernel would round differently.  tests/test_gpu_fused_post_smoothing.py holds
// the two to the same bits.
constexpr int kPjRing = 4;
constexpr int kPjArr = 9;  // x_old (2), exx, eyy, 1/ezz of the raw row; rhs (2) and omega/diag (2) of sweep 1's output row
__host__ __device__ inline size_t pj_stage_floats(int W, int nyc) { return (size_t)kPjArr * 2 * W + 4 * (size_t)((nyc + 3) & ~3); }
inline size_t pj_smem(int W, int nyc) { return kPjRing * pj_stage_floats(W, nyc) * sizeof(float); }

// x + P e_c at one fine value out of the coarse rows c0 (I0) and c1 (I1)
__device__ __forceinline__ float pj_prolong(float x, float wx0, float wx1, const float *c0, const float *c1, int J0, int J1, float wy0,
                                            float wy1) {
  return __fadd_rn(x, __fmaf_rn(wx0, __fmaf_rn(wy0, c0[J0], __fmul_rn(wy1, c0[J1])), __fmul_rn(wx1, __fmaf_rn(wy0, c1[J0], __fmul_rn(wy1, c1[J1])))));
}

// u = -(1/ezz (b0 a1 + bm a0 + yb0 b1 + ybm bl)) and t = f0 v21 + f1 v22 - yf0 v11 - yf1 v11' of the march
__device__ __forceinline__ float pj_u(float ie, float b0, float a1, float bm, float a0, float yb0, float b1, float ybm, float bl) {
  return -__fmul_rn(ie, __fmaf_rn(ybm, bl, __fmaf_rn(yb0, b1, __fmaf_rn(b0, a1, __fmul_rn(bm, a0)))));
}
__device__ __forceinline__ float pj_t(float f0, float v21, float f1, float v22, float yf0, float v11, float yf1, float v11r) {
  return __fmaf_rn(-yf1, v11r, __fmaf_rn(-yf0, v11, __fmaf_rn(f0, v21, __fmul_rn(f1, v22))));
}
// the stored-diagonal sweep's output pair of row k: x + (omega/diag) (rhs - (A - sigma) x), both components
__device__ __forceinline__ void pj_sweep(const RowCoef<float> &xc, float2 yf0, float2 yf1, float2 yb0, float2 ybm, float sg, float2 u0,
                                         float2 u1, float ur, float2 t0, float2 tm, float tl, float2 a0, float2 b0, float2 v10,
                                         float2 v20, float2 cr1, float2 cr2, float2 cd1, float2 cd2, float2 &w1, float2 &w2) {
  const float p1x = __fmaf_rn(xc.f0, u0.x, __fmul_rn(xc.f1, u1.x)), p1y = __fmaf_rn(xc.f0, u0.y, __fmul_rn(xc.f1, u1.y));
  const float p2x = __fmaf_rn(yf1.x, u0.y, __fmul_rn(yf0.x, u0.x)), p2y = __fmaf_rn(yf0.y, u0.y, __fmul_rn(yf1.y, ur));
  const float c1x = __fsub_rn(__fmaf_rn(yb0.x, t0.x, __fmul_rn(ybm.x, tl)), a0.x), c1y = __fsub_rn(__fmaf_rn(yb0.y, t0.y, __fmul_rn(ybm.y, t0.x)), a0.y);
  const float c2x = __fadd_rn(__fmaf_rn(xc.bm, tm.x, __fmul_rn(xc.b0, t0.x)), b0.x), c2y = __fadd_rn(__fmaf_rn(xc.bm, tm.y, __fmul_rn(xc.b0, t0.y)), b0.y);
  const float o1x = __fmaf_rn(-sg, v10.x, __fadd_rn(p1x, c1x)), o1y = __fmaf_rn(-sg, v10.y, __fadd_rn(p1y, c1y));
  const float o2x = __fmaf_rn(-sg, v20.x, __fsub_rn(p2x, c2x)), o2y = __fmaf_rn(-sg, v20.y, __fsub_rn(p2y, c2y));
  w1 = make_float2(__fmaf_rn(cd1.x, __fsub_rn(cr1.x, o1x), v10.x), __fmaf_rn(cd1.y, __fsub_rn(cr1.y, o1y), v10.y));
  w2 = make_float2(__fmaf_rn(cd2.x, __fsub_rn(cr2.x, o2x), v20.x), __fmaf_rn(cd2.y, __fsub_rn(cr2.y, o2y), v20.y));
}

__global__ void __launch_bounds__(kM2MaxW, 2) stencil_prolong_jacobi2_kernel(StencilArgs<float, float> a, int rows) {
  using T = float;
  using V = float2;
  __shared__ T sB[2][2][kM2MaxW + 2], sV[2][2][kM2MaxW + 2], sU[2][2][kM2MaxW + 2], sTt[2][2][kM2MaxW + 2];  // [sweep][buffer]
  __shared__ RowCoef<T> sX[kM2MaxSteps + 3];  // coefficients of rows k0 - 2 ..
  __shared__ int4 sPi[kM2MaxSteps];           // coarse rows of raw row k0 + 2 + j: x-edge I0, I1, x-node I0, I1
  __shared__ float4 sPw[kM2MaxSteps];         // and their weights
  __shared__ __align__(8) unsigned long long sBar[kPjRing];
  extern __shared__ __align__(128) unsigned char m2_ring_raw[];  // [kPjRing][kPjArr][W] float2, then [4][nyc rounded to 4] floats
  T *ring = reinterpret_cast<T *>(m2_ring_raw);

  const TransferArgs &tr = *a.tr;
  const int nx = a.nx, ny = a.ny, nyc = tr.nyc;
  const int nycp = (nyc + 3) & ~3;
  const int W = blockDim.x;
  const unsigned N = (unsigned)nx * (unsigned)ny;
  const size_t Nc = (size_t)tr.nxc * nyc;
  const int b = blockIdx.z;
  const int c = threadIdx.x;
  const int npairs = ny >> 1;
  const int gj = 2 * c;
  const bool colv = c < npairs;
  const int i0 = blockIdx.y * rows;
  const int iend = (i0 + rows < nx) ? i0 + rows : nx;
  const int k0 = i0 - 4;
  const int nsteps = rows + 6;
  const int raw_lo = max(i0 - 2, 0), raw_hi = min(iend + 1, nx - 1);  // rows the prolongation forms
  const int s1_lo = max(i0 - 1, 0), s1_hi = min(iend, nx - 1);       // rows sweep 1 outputs
  const size_t stf = pj_stage_floats(W, nyc);
  const T *x1 = a.x + (size_t)b * 2 * N, *x2 = x1 + N;
  const T *fb = a.fields + a.field_bstride * b;
  const T *exx = fb, *eyy = fb + N, *iez = fb + 2 * (size_t)N;
  const T *cx = a.cx + (size_t)b * 4 * nx, *cy = a.cy + (size_t)b * 4 * ny;
  const T *r1 = a.rhs + (size_t)b * 2 * N, *r2 = r1 + N;
  const T *d1 = a.dinv + (size_t)b * 2 * N, *d2 = d1 + N;
  const T *cb = a.coarse + (size_t)b * 2 * Nc;  // coarse correction, component 0 (component 1 at + Nc)
  T *y1 = a.y + (size_t)b * 2 * N, *y2 = y1 + N;
  const T zT = 0.0f;
  const V zV = {zT, zT};
  const unsigned nbytes = (unsigned)npairs * (unsigned)sizeof(V);

  // lanes 0 .. kPjArr-1 of warp 0 each own one array (bulk copies); every thread copies its share of the four coarse rows and
  // arrives on the stage's barrier (W + 1 arrivals per phase: lane 0's expect_tx and one per thread)
  const T *my_arr = nullptr;
  if (c == 0) my_arr = x1; else if (c == 1) my_arr = x2; else if (c == 2) my_arr = exx; else if (c == 3) my_arr = eyy; else if (c == 4) my_arr = iez;
  else if (c == 5) my_arr = r1; else if (c == 6) my_arr = r2; else if (c == 7) my_arr = d1; else if (c == 8) my_arr = d2;
  auto issue = [&](int jj) {
    const int stage = jj & (kPjRing - 1);
    const int gr = k0 + jj + 2, go = k0 + jj;
    const bool rawv = gr >= raw_lo && gr <= raw_hi;
    const bool outv = go >= s1_lo && go <= s1_hi;
    unsigned long long *bar = &sBar[stage];
    T *st = ring + stage * stf;
    if (c == 0) mbar_expect_tx(bar, ((rawv ? 5u : 0u) + (outv ? 4u : 0u)) * nbytes);
    if (c < kPjArr && (c < 5 ? rawv : outv)) bulk_g2s(st + (size_t)c * 2 * W, my_arr + (size_t)(c < 5 ? gr : go) * ny, nbytes, bar);
    if (rawv) {
      const int4 pi = sPi[jj];
      const int ci[4] = {pi.x, pi.y, pi.z, pi.w};
      T *cs = st + (size_t)kPjArr * 2 * W;
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        const T *src = cb + (r >> 1) * Nc + (size_t)ci[r] * nyc;
        for (int e = c; e < nyc; e += W) cp_async4(cs + r * nycp + e, src + e);
      }
    }
    cp_async_arrive(bar);
  };

  if (c == 0) {
#pragma unroll
    for (int s = 0; s < kPjRing; ++s) mbar_init(&sBar[s], W + 1);
    mbar_fence_init();
  }
  for (int r = c; r < nsteps + 3; r += W) {  // coefficients of rows k0 - 2 .. k0 + nsteps
    const int gi = k0 - 2 + r;
    RowCoef<T> rc;
    rc.f0 = rc.f1 = rc.b0 = rc.bm = zT;
    if (gi >= 0 && gi < nx) { rc.f0 = __ldg(cx + gi); rc.f1 = __ldg(cx + nx + gi); rc.b0 = __ldg(cx + 2 * nx + gi); rc.bm = __ldg(cx + 3 * nx + gi); }
    sX[r] = rc;
  }
  for (int r = c; r < nsteps; r += W) {  // prolongation rows of the raw rows k0 + 2 ..
    const int gi = k0 + 2 + r;
    int4 pi = make_int4(0, 0, 0, 0);
    float4 pw = make_float4(0.f, 0.f, 0.f, 0.f);
    if (gi >= 0 && gi < nx) {
      pi = make_int4(__ldg(tr.xe.p_i0 + gi), __ldg(tr.xe.p_i1 + gi), __ldg(tr.xn.p_i0 + gi), __ldg(tr.xn.p_i1 + gi));
      pw = make_float4(__ldg(tr.xe.p_w0f + gi), __ldg(tr.xe.p_w1f + gi), __ldg(tr.xn.p_w0f + gi), __ldg(tr.xn.p_w1f + gi));
    }
    sPi[r] = pi;
    sPw[r] = pw;
  }
  for (int p = 0; p < 2; ++p)
    for (int s = 0; s < 2; ++s) {
      sB[p][s][c + 1] = zT; sV[p][s][c + 1] = zT; sU[p][s][c + 1] = zT; sTt[p][s][c + 1] = zT;
      if (c < 2) {
        const int e = c == 0 ? 0 : W + 1;
        sB[p][s][e] = zT; sV[p][s][e] = zT; sU[p][s][e] = zT; sTt[p][s][e] = zT;
      }
    }
  V yf0 = zV, yf1 = zV, yb0 = zV, ybm = zV;
  // y-lists of the pair's two columns: y-node lists for component 0, y-edge lists for component 1; the coarse column pair
  // J0 | J1 << 16 per fine column (nyc < 2^16) keeps the two sweeps' pipelines within 128 registers
  int2 jn = make_int2(0, 0), je = jn;
  V wn0 = zV, wn1 = zV, we0 = zV, we1 = zV;
  if (colv) {
    yf0 = ldg2(cy + gj); yf1 = ldg2(cy + ny + gj); yb0 = ldg2(cy + 2 * ny + gj); ybm = ldg2(cy + 3 * ny + gj);
    const int2 jn0 = __ldg(reinterpret_cast<const int2 *>(tr.yn.p_i0 + gj)), jn1 = __ldg(reinterpret_cast<const int2 *>(tr.yn.p_i1 + gj));
    const int2 je0 = __ldg(reinterpret_cast<const int2 *>(tr.ye.p_i0 + gj)), je1 = __ldg(reinterpret_cast<const int2 *>(tr.ye.p_i1 + gj));
    jn = make_int2(jn0.x | jn1.x << 16, jn0.y | jn1.y << 16);
    je = make_int2(je0.x | je1.x << 16, je0.y | je1.y << 16);
    wn0 = ldg2(tr.yn.p_w0f + gj); wn1 = ldg2(tr.yn.p_w1f + gj); we0 = ldg2(tr.ye.p_w0f + gj); we1 = ldg2(tr.ye.p_w1f + gj);
  }
  const bool mask_col0 = tr.mask_y && gj == 0 && ny > 1;  // component 0, fine column 0
  const bool mask_row0 = tr.mask_x && nx > 1;              // component 1, fine row 0
  const T sg = __ldg(a.sigma + b);
  __syncthreads();  // barriers initialised, row tables and exchange rows in place
#pragma unroll
  for (int s = 0; s < kPjRing; ++s)
    if (s < nsteps) issue(s);

  // sweep 1 (raw rows: x_old + P e_c) and sweep 2 (raw rows: sweep 1's output), each the register pipeline of the march
  V a1 = zV, b1 = zV, v11 = zV, v21 = zV, a0 = zV, b0 = zV, v10 = zV, v20 = zV, ie1 = zV;
  V u0 = zV, t0 = zV, tm = zV;
  V ha1 = zV, hb1 = zV, hv11 = zV, hv21 = zV, ha0 = zV, hb0 = zV, hv10 = zV, hv20 = zV, hie1 = zV;
  V hu0 = zV, ht0 = zV, htm = zV;
  RowCoef<T> xc = sX[2], hxc = sX[0];  // coefficients of the output rows k (sweep 1) and k - 2 (sweep 2)

  // two-fold unroll (the exchange buffer index stays a constant): unrolled six-fold like the kernels above it spills at 128 registers
  for (int j0 = 0; j0 < nsteps; j0 += 2) {
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const int j = j0 + u, k = k0 + j;
      const int s = u & 1, sp = s ^ 1;
      const int stage = j & (kPjRing - 1);
      mbar_wait(&sBar[stage], (unsigned)(j / kPjRing) & 1u);
      const T *stT = ring + stage * stf;
      const V *st = reinterpret_cast<const V *>(stT);
      const V *sth = reinterpret_cast<const V *>(ring + ((j - 2) & (kPjRing - 1)) * stf);  // stage of step j - 2
      // stage 0: raw row k+2 = x_old + P e_c
      const int gr = k + 2;
      V v12 = zV, v22 = zV, ex2 = zV, ey2 = zV, ie2 = zV;
      if (gr >= raw_lo && gr <= raw_hi && colv) {
        v12 = st[0 * W + c]; v22 = st[1 * W + c]; ex2 = st[2 * W + c]; ey2 = st[3 * W + c]; ie2 = st[4 * W + c];
        const float4 pw = sPw[j];
        const T *cs = stT + (size_t)kPjArr * 2 * W;
        if (!mask_col0) v12.x = pj_prolong(v12.x, pw.x, pw.y, cs, cs + nycp, jn.x & 0xffff, jn.x >> 16, wn0.x, wn1.x);
        v12.y = pj_prolong(v12.y, pw.x, pw.y, cs, cs + nycp, jn.y & 0xffff, jn.y >> 16, wn0.y, wn1.y);
        if (!(mask_row0 && gr == 0)) {
          v22.x = pj_prolong(v22.x, pw.z, pw.w, cs + 2 * nycp, cs + 3 * nycp, je.x & 0xffff, je.x >> 16, we0.x, we1.x);
          v22.y = pj_prolong(v22.y, pw.z, pw.w, cs + 2 * nycp, cs + 3 * nycp, je.y & 0xffff, je.y >> 16, we0.y, we1.y);
        }
      }
      // stage 1: sweep 1, output row k
      V a2, b2;
      a2.x = __fmul_rn(ex2.x, v12.x); a2.y = __fmul_rn(ex2.y, v12.y);
      b2.x = __fmul_rn(ey2.x, v22.x); b2.y = __fmul_rn(ey2.y, v22.y);
      sB[0][s][c + 1] = b2.y;
      sV[0][s][c + 1] = v12.x;
      const T bl = sB[0][sp][c], v1r = sV[0][sp][c + 2];
      const RowCoef<T> xn = sX[j + 3];
      V u1, t1;
      u1.x = pj_u(ie1.x, xn.b0, a1.x, xn.bm, a0.x, yb0.x, b1.x, ybm.x, bl);
      u1.y = pj_u(ie1.y, xn.b0, a1.y, xn.bm, a0.y, yb0.y, b1.y, ybm.y, b1.x);
      t1.x = pj_t(xn.f0, v21.x, xn.f1, v22.x, yf0.x, v11.x, yf1.x, v11.y);
      t1.y = pj_t(xn.f0, v21.y, xn.f1, v22.y, yf0.y, v11.y, yf1.y, v1r);
      sU[0][s][c + 1] = u1.x;
      sTt[0][s][c + 1] = t1.y;
      const bool s1v = colv && k >= s1_lo && k <= s1_hi;
      V w1 = zV, w2 = zV;  // sweep 1 at row k (zero outside the rows sweep 2 reads, as its raw rows outside the grid)
      if (s1v) {
        const T ur = sU[0][sp][c + 2], tl = sTt[0][sp][c];
        pj_sweep(xc, yf0, yf1, yb0, ybm, sg, u0, u1, ur, t0, tm, tl, a0, b0, v10, v20, st[5 * W + c], st[6 * W + c], st[7 * W + c],
                 st[8 * W + c], w1, w2);
      }
      // stage 2: sweep 2 with row k of sweep 1 as its newest row, output row k - 2
      V hex2 = zV, hey2 = zV, hie2 = zV;
      if (s1v) { hex2 = sth[2 * W + c]; hey2 = sth[3 * W + c]; hie2 = sth[4 * W + c]; }
      V ha2, hb2;
      ha2.x = __fmul_rn(hex2.x, w1.x); ha2.y = __fmul_rn(hex2.y, w1.y);
      hb2.x = __fmul_rn(hey2.x, w2.x); hb2.y = __fmul_rn(hey2.y, w2.y);
      sB[1][s][c + 1] = hb2.y;
      sV[1][s][c + 1] = w1.x;
      const T hbl = sB[1][sp][c], hv1r = sV[1][sp][c + 2];
      const RowCoef<T> hxn = sX[j + 1];
      V hu1, ht1;
      hu1.x = pj_u(hie1.x, hxn.b0, ha1.x, hxn.bm, ha0.x, yb0.x, hb1.x, ybm.x, hbl);
      hu1.y = pj_u(hie1.y, hxn.b0, ha1.y, hxn.bm, ha0.y, yb0.y, hb1.y, ybm.y, hb1.x);
      ht1.x = pj_t(hxn.f0, hv21.x, hxn.f1, w2.x, yf0.x, hv11.x, yf1.x, hv11.y);
      ht1.y = pj_t(hxn.f0, hv21.y, hxn.f1, w2.y, yf0.y, hv11.y, yf1.y, hv1r);
      sU[1][s][c + 1] = hu1.x;
      sTt[1][s][c + 1] = ht1.y;
      const int ko = k - 2;
      if (colv && ko >= i0 && ko < iend) {
        const T ur = sU[1][sp][c + 2], tl = sTt[1][sp][c];
        V z1, z2;
        pj_sweep(hxc, yf0, yf1, yb0, ybm, sg, hu0, hu1, ur, ht0, htm, tl, ha0, hb0, hv10, hv20, sth[5 * W + c], sth[6 * W + c],
                 sth[7 * W + c], sth[8 * W + c], z1, z2);
        const unsigned g = (unsigned)ko * (unsigned)ny + (unsigned)gj;
        stg2(y1 + g, z1.x, z1.y);
        stg2(y2 + g, z2.x, z2.y);
      }
      tm = t0; t0 = t1; u0 = u1;
      a0 = a1; b0 = b1; v10 = v11; v20 = v21; a1 = a2; b1 = b2; v11 = v12; v21 = v22;
      ie1 = ie2;
      xc = xn;
      htm = ht0; ht0 = ht1; hu0 = hu1;
      ha0 = ha1; hb0 = hb1; hv10 = hv11; hv20 = hv21; ha1 = ha2; hb1 = hb2; hv11 = w1; hv21 = w2;
      hie1 = hie2;
      hxc = hxn;
      __syncthreads();
      // every thread is done with the stage of step j - 2: refill it with the rows of step j + 2
      if (j >= 2 && j + 2 < nsteps) issue(j + 2);
    }
  }
}

}  // namespace b200ms
