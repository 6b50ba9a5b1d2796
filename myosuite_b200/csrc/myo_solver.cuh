// myo_solver.cuh -- constraint assembly, primal Newton solver and semi-implicit Euler (one env per warp).
// Semantics: MuJoCo's soft-constraint model (SURVEY.md Appendix A.5): rows = joint equalities, joint
// limits, pyramidal/frictionless contacts; cost 1/2 (a-a0)'M(a-a0) + sum_i s_i(J_i a - aref_i);
// Newton with exact line search on H = M + J' D_active J (register/shuffle Cholesky of the dense packed H; tree-sparse L'DL when no contact is active).
#pragma once
#include "myo_device.cuh"

// scratch views (stage 3/4): shared-space pointer expressions (m.s_* are offsets from the warp base)
#define S_H SCR(s_H)
#define S_con SCR(s_con)
// Contact Jacobian rows are STORED as the upper 48 bits of the f64 value (sign, exponent, 36 mantissa bits: a u32 high word and a u16 middle
// word, rounded to nearest), i.e. 1.5e-11 relative per entry; the arithmetic stays f64 and no conversion instruction is needed to rebuild
// the double.  Measured round 2: f32 storage (6e-8 per entry) moved qacc by up to 9e-5 relative on stiff multi-contact hand states -- beyond
// the north-star's 1e-5 -- while f64 storage does not leave room for 14 env-warps per SM.  -DMYO_F64_ROWS stores plain doubles (the
// verification build, abi.lib("f64rows")).  The regularisers D are f64 in both builds: one per equality / limit row and ONE per contact (the
// rows of a contact share it), found through the byte map S_drow.
struct JacRef {
#ifdef MYO_F64_ROWS
  double* p;
  __device__ __forceinline__ double operator[](int i) const { return p[i]; }
  __device__ __forceinline__ double put(int i, double v) const { p[i] = v; return v; }
  __device__ __forceinline__ JacRef operator+(int k) const { return JacRef{p + k}; }
#else
  unsigned* h; unsigned short* l;
  __device__ __forceinline__ double operator[](int i) const { return __hiloint2double((int)h[i], (int)((unsigned)l[i] << 16)); }
  __device__ __forceinline__ double put(int i, double v) const {            // stores and returns the rounded value
    const unsigned long long b = (unsigned long long)__double_as_longlong(v) + 0x8000ull; const unsigned hi = (unsigned)(b >> 32), mid = (unsigned)(b >> 16) & 0xffffu;
    h[i] = hi; l[i] = (unsigned short)mid; return __hiloint2double((int)hi, (int)(mid << 16)); }
  __device__ __forceinline__ JacRef operator+(int k) const { return JacRef{h + k, l + k}; }
#endif
};
#ifdef MYO_F64_ROWS
#define JAC_BYTES 8
#define S_jac(c) (JacRef{SCR(s_conJ) + (c)*3*m.maxpath})
#else
#define JAC_BYTES 6
#define S_jac(c) (JacRef{(unsigned*)SCR(s_conJ) + (c)*3*m.maxpath, (unsigned short*)((unsigned*)SCR(s_conJ) + 3*m.maxpath*m.maxcon) + (c)*3*m.maxpath})
#endif
#define S_D SCR(s_efD)
#define S_DCON(c) (m.neq + m.nlimrow + (c))      // index of contact c's regulariser in S_D
#define S_aref SCR(s_efA)
#define S_jar SCR(s_efR)
#define S_jv SCR(s_efV)
#define S_a SCR(s_va)
#define S_g SCR(s_vg)
#define S_p SCR(s_vp)
#define S_Ma SCR(s_vMa)
#define S_Mp SCR(s_vMp)
#define S_eqJ SCR(s_eqJ)
#define S_Hs SCR(s_Hs)
#define S_LD SCR(s_LD)
#define S_Dinv SCR(s_Dinv)
// integer records of the contact / row lists (S_cpair is defined in myo_device.cuh: the colliders write it)
#define S_cmask ((unsigned long long*)SCR(s_icon))   // contact -> bit mask of the dofs on its path (the Jacobian's non-zero columns, ascending)
#define S_crown ((int*)(SCR(s_icon) + m.maxcon))     // contact -> first efc row | number of rows << 12 | rank in model pair order << 16
#define CROW(rn) ((rn) & 0xfff)
#define CNR(rn) (((rn) >> 12) & 7)
#define CRANK(rn) ((rn) >> 16)
#define S_lrow (S_cpair + m.maxcon)            // limit row descriptors, int16: dof | side << 8
#define S_drow ((unsigned char*)(S_lrow + m.nlimrow + 4))      // constraint row -> index of its regulariser in S_D

__device__ __forceinline__ double impedance(const double* si, double pos, double margin) {
  if (si[0] == si[1] || si[2] <= MYO_MINVAL) return 0.5*(si[0]+si[1]);
  double x = fabs((pos-margin)*m_rcp(si[2]));
  if (x >= 1 || x <= 0) return x >= 1 ? si[1] : si[0];
  double y;
  if (si[4] == 1) y = x;
  else if (si[4] == 2) y = x <= si[3] ? x*x*m_rcp(si[3]) : 1-(1-x)*(1-x)*m_rcp(1-si[3]);   // the default power, without pow()
  else if (x <= si[3]) y = pow(x, si[4])/pow(si[3], si[4]-1);
  else y = 1-pow(1-x, si[4])/pow(1-si[3], si[4]-1);
  return si[0]+y*(si[1]-si[0]); }

// y = M x using the per-row non-zero lists
template <class MD> __device__ __forceinline__ void mul_M(const MD& m, const Warp w, double* y, const double* x) {
  const idx_t* radr = CI(PROW_adr); const idx_t* rcol = CI(PROW_col); const idx_t* ridx = CI(PROW_idx);
  for (int i = w.lane; i < m.nv; i += 32) { double s = 0; for (int e = radr[i]; e < radr[i+1]; e++) s += W_(qM)[ridx[e]]*x[rcol[e]]; y[i] = s; } }

// out[r] = (J x)_r for every constraint row
template <class MD> __device__ void rows_apply(const MD& m, const Warp w, const double* x, double* out) {
  SHARED_PTR(x); SHARED_PTR(out);
  const idx_t* eq = CI(PEQ); const int nlimrow = WI_(nlimrow), ncon = WI_(ncon);
  for (int e = w.lane; e < m.neq; e += 32) { double v = x[eq[PEQ_ISTRIDE*e+1]]; if (eq[PEQ_ISTRIDE*e+3] >= 0) v += S_eqJ[e]*x[eq[PEQ_ISTRIDE*e+3]]; out[e] = v; }
  for (int r = w.lane; r < nlimrow; r += 32) { int dsc = S_lrow[r]; double sg = (dsc >> 8) & 1 ? -1.0 : 1.0; out[m.neq + r] = sg*x[dsc & 0xff]; }
  const idx_t* pr = CI(PPAIR); const idx_t* path = CI(PPATH);
  for (int c = w.lane; c < ncon; c += 32) { const int rn = S_crown[c], nr = CNR(rn); if (!nr) continue;
    const idx_t* q = pr + PPAIR_ISTRIDE*S_cpair[c]; const JacRef J = S_jac(c); double n = 0, t1 = 0, t2 = 0;
    for (int e = 0; e < q[4]; e++) { double xv = x[path[q[3]+e] >> 1]; n += J[3*e]*xv; t1 += J[3*e+1]*xv; t2 += J[3*e+2]*xv; }
    int rb = CROW(rn);
    if (nr == 1) out[rb] = n;
    else { out[rb] = n+t1; out[rb+1] = n-t1; out[rb+2] = n+t2; out[rb+3] = n-t2; } }
}

// vec[d] += sum_r J[r][d] * wgt[r]  (wgt already includes D and the active mask; wgt is DESTROYED: the rows of a contact are folded into its
// normal / tangent weights in place).  Contacts are GATHERED: lane d owns vec[d] and walks the contact list, testing its bit in each contact's
// path mask; the position of d in the contact's Jacobian is the number of lower bits set (paths list dofs in ascending order).  No lane
// waits for another contact's rows: round 1 looped over the contacts with a warp sync and <= 8 busy lanes per contact.
template <class MD> __device__ void rows_applyT_add(const MD& m, const Warp w, double* wgt, double* vec) {
  SHARED_PTR(wgt); SHARED_PTR(vec);
  const idx_t* eq = CI(PEQ); const int nlimrow = WI_(nlimrow), ncon = WI_(ncon);
  if (w.lane == 0) for (int e = 0; e < m.neq; e++) { vec[eq[PEQ_ISTRIDE*e+1]] += wgt[e]; if (eq[PEQ_ISTRIDE*e+3] >= 0) vec[eq[PEQ_ISTRIDE*e+3]] += S_eqJ[e]*wgt[e]; }
  __syncwarp();
  for (int pass = 0; pass < 2; pass++) {
    for (int r = w.lane; r < nlimrow; r += 32) { int dsc = S_lrow[r]; int neg = (dsc >> 8) & 1; if (neg == pass) vec[dsc & 0xff] += (neg ? -1.0 : 1.0)*wgt[m.neq + r]; }
    __syncwarp(); }
  for (int c = w.lane; c < ncon; c += 32) { const int rn = S_crown[c], nr = CNR(rn), rb = CROW(rn);      // fold the pyramid edges: (wn, w1, w2) into wgt[rb .. rb+2]
    if (nr == 4) { const double a0 = wgt[rb], a1 = wgt[rb+1], a2 = wgt[rb+2], a3 = wgt[rb+3];
      wgt[rb] = a0+a1+a2+a3; wgt[rb+1] = a0-a1; wgt[rb+2] = a2-a3; } }
  __syncwarp();
  for (int d = w.lane; d < m.nv; d += 32) { double acc = 0; const unsigned long long below = (1ull << d) - 1;
    for (int c = 0; c < ncon; c++) { const unsigned long long mk = S_cmask[c];
      if ((mk >> d) & 1) { const int rn = S_crown[c], nr = CNR(rn), rb = CROW(rn); const JacRef J = S_jac(c) + 3*__popcll(mk & below);
        if (nr == 4) acc += J[0]*wgt[rb] + J[1]*wgt[rb+1] + J[2]*wgt[rb+2]; else if (nr == 1) acc += J[0]*wgt[rb]; } }
    vec[d] += acc; }
  __syncwarp();
}

// ------------------------------------------------------------------ constraint assembly
// residual of joint equality record c (PEQ_d) at qpos: q1 - q1_0 - poly(q2 - q2_0), or q1 - q1_0 - c[0] without a second joint (q2 < 0);
// deriv = d poly / d q2 (0 without a second joint), so that the row's Jacobian is 1 at d1 and -deriv at d2.  The same expressions as the
// equality rows of phase_constraints below, which keeps its own inline copy: routing it through this helper reorders the step kernels'
// machine code.
__device__ __forceinline__ double eq_residual(const double* c, const double* qpos, int q1, int q2, double& deriv) {
  const double pos0 = qpos[q1]-c[5];
  if (q2 >= 0) { double x = qpos[q2]-c[6]; deriv = c[1]+x*(2*c[2]+x*(3*c[3]+x*4*c[4])); return pos0-(c[0]+x*(c[1]+x*(c[2]+x*(c[3]+x*c[4])))); }
  deriv = 0; return pos0-c[0]; }

template <class MD> __device__ void phase_constraints(const MD& m, const Warp w) {
  // joint equalities (always active)
  const idx_t* eq = CI(PEQ); const double* eqd = CD(PEQ_d);
  for (int e = w.lane; e < m.neq; e += 32) { const double* c = eqd + e*PEQ_STRIDE; int q1 = eq[PEQ_ISTRIDE*e], d1 = eq[PEQ_ISTRIDE*e+1], q2 = eq[PEQ_ISTRIDE*e+2], d2 = eq[PEQ_ISTRIDE*e+3];
    double pos0 = W_(qpos)[q1]-c[5], cpos, deriv = 0, vel = W_(qvel)[d1];
    if (q2 >= 0) { double x = W_(qpos)[q2]-c[6]; cpos = pos0-(c[0]+x*(c[1]+x*(c[2]+x*(c[3]+x*c[4])))); deriv = c[1]+x*(2*c[2]+x*(3*c[3]+x*4*c[4])); vel -= deriv*W_(qvel)[d2]; }
    else cpos = pos0-c[0];
    S_eqJ[e] = -deriv;
    double imp = impedance(c+10, cpos, 0), R = fmax(MYO_MINVAL, (1-imp)*c[7]*m_rcp(imp));
    S_D[e] = m_rcp(R); S_drow[e] = (unsigned char)e; S_aref[e] = -c[9]*vel - c[8]*imp*cpos; }
  // joint limits (one-sided)
  const idx_t* lim = CI(PLIM); const double* __restrict__ limd = GD(PLIM_d); int nrow = 0;      // (cold table: one 12-double record per limited joint, read once per substep)
  for (int base = 0; base < m.nlim; base += 32) { int l = base + w.lane; bool lo = false, hi = false; double dlo = 0, dhi = 0; double c[PLIM_STRIDE]; for (int k = 0; k < PLIM_STRIDE; k++) c[k] = LDC(limd + (l < m.nlim ? l : 0)*PLIM_STRIDE + k); int d = 0;
    if (l < m.nlim) { d = lim[2*l]; double q = W_(qpos)[lim[2*l+1]]; dlo = q-c[0]; dhi = c[1]-q; lo = dlo < c[2]; hi = dhi < c[2]; }
    unsigned m0 = __ballot_sync(FULL, lo), m1 = __ballot_sync(FULL, hi), lt = (1u << w.lane)-1; int idx = nrow + __popc(m0 & lt) + __popc(m1 & lt);
    for (int side = 0; side < 2; side++) { if (!(side ? hi : lo)) continue;
      double dist = side ? dhi : dlo, sg = side ? -1.0 : 1.0; int r = m.neq + idx; idx++;
      S_lrow[r - m.neq] = (idx_t)(d | (side << 8));
      double imp = impedance(c+6, dist, c[2]), R = fmax(MYO_MINVAL, (1-imp)*c[3]*m_rcp(imp));
      S_D[r] = m_rcp(R); S_drow[r] = (unsigned char)r; S_aref[r] = -c[5]*sg*W_(qvel)[d] - c[4]*imp*(dist-c[2]); }
    nrow += __popc(m0) + __popc(m1); }
  WI_(nlimrow) = nrow;
  // contacts: Jacobian over the dofs between the two bodies, regulariser, reference acceleration.
  // The contact list holds two runs (analytic colliders [0, na), ellipsoid colliders [na, ncon)), each in model pair order.  Records stay
  // where the colliders put them; what follows MuJoCo's contact order is the RANK of each contact (reported by the parity taps) and the
  // numbering of the constraint rows, which are assigned in rank order.
  const idx_t* pr = CI(PPAIR); const double* pd = CD(PPAIR_d); const idx_t* path = CI(PPATH);
  int rowbase = m.neq + nrow; const int ncon = WI_(ncon), na = WI_(na);
  int* key = (int*)SCR(s_conJ);                              // scratch: the Jacobians are written after the last read of the keys
  for (int c = w.lane; c < ncon; c += 32) key[c] = pr[PPAIR_ISTRIDE*S_cpair[c] + 7];
  __syncwarp();
  int nrs[2] = {0, 0}, rank[2] = {0, 0}, rbs[2] = {0, 0};
  #pragma unroll
  for (int s = 0; s < 2; s++) { const int c = w.lane + 32*s;
    if (c < ncon) { const idx_t* q = pr + PPAIR_ISTRIDE*S_cpair[c]; const double* P = pd + q[6]*PPAIR_STRIDE;
      nrs[s] = (S_con[c*CON_STRIDE] < P[0]-P[1]) ? (q[2] == 1 ? 1 : 4) : 0;
      const int k = key[c]; int cnt = 0;
      if (c < na) { for (int q2 = na; q2 < ncon; q2++) cnt += key[q2] < k; rank[s] = c + cnt; }
      else { for (int q2 = 0; q2 < na; q2++) cnt += key[q2] < k; rank[s] = (c - na) + cnt; }
      S_crown[rank[s]] = nrs[s]; } }
  __syncwarp();
  #pragma unroll
  for (int s = 0; s < 2; s++) { const int k = w.lane + 32*s; const int v = k < ncon ? S_crown[k] : 0; int incl = v;   // inclusive warp scan in rank order
    #pragma unroll
    for (int o = 1; o < 32; o <<= 1) { int t = __shfl_up_sync(FULL, incl, o); if (w.lane >= o) incl += t; }
    if (k < ncon) S_crown[k] = rowbase + incl - v;
    rowbase += __shfl_sync(FULL, incl, 31); }
  __syncwarp();
  #pragma unroll
  for (int s = 0; s < 2; s++) { const int c = w.lane + 32*s; if (c < ncon) rbs[s] = S_crown[rank[s]]; }
  __syncwarp();
  #pragma unroll
  for (int s = 0; s < 2; s++) { const int c = w.lane + 32*s, nr = nrs[s], rb = rbs[s];
    if (c < ncon) S_crown[c] = rb | (nr << 12) | (rank[s] << 16);
    if (c < ncon && nr) { const idx_t* q = pr + PPAIR_ISTRIDE*S_cpair[c]; const double* P = pd + q[6]*PPAIR_STRIDE; const double* cd = S_con + c*CON_STRIDE;
      const double* pos = cd + 1; double f[9]; for (int k = 0; k < 6; k++) f[k] = cd[4+k]; cross3(f+6, f, f+3); const JacRef J = S_jac(c); double vn = 0, v1 = 0, v2 = 0;
      unsigned long long mk = 0; const double mu1 = P[2], mu2 = P[3];
      for (int e = 0; e < q[4]; e++) { int code = path[q[3]+e], d = code >> 1; double sg = (code & 1) ? 1.0 : -1.0, cv[3]; dof_point_vel(m, w, d, pos, cv); mk |= 1ull << d;
        const double jn = J.put(3*e, sg*dot3(f, cv)), j1 = J.put(3*e+1, sg*mu1*dot3(f+3, cv)), j2 = J.put(3*e+2, sg*mu2*dot3(f+6, cv));      // tangents stored times mu: the pyramid edges are n +- mu t
        double qd = W_(qvel)[d]; vn += jn*qd; v1 += j1*qd; v2 += j2*qd; }      // (aref from the stored Jacobian: consistent with J v in the solver)
      S_cmask[c] = mk;
      double dist = cd[0], inc = P[0]-P[1], imp = impedance(P+7, dist, inc), K = P[5], B = P[6], tran = LDC(GD(PPAIR_tran) + S_cpair[c]);
      const unsigned char dc = (unsigned char)S_DCON(c);
      if (nr == 1) { double R = fmax(MYO_MINVAL, (1-imp)*tran*m_rcp(imp)); S_D[dc] = m_rcp(R); S_drow[rb] = dc; S_aref[rb] = -B*vn - K*imp*(dist-inc); }
      else { double R0 = fmax(MYO_MINVAL, (1-imp)*(tran+mu1*mu1*tran)*m_rcp(imp)), Rpy = 2*mu1*mu1*R0, Dv = m_rcp(Rpy), kp = K*imp*(dist-inc);
        S_D[dc] = Dv; S_drow[rb] = S_drow[rb+1] = S_drow[rb+2] = S_drow[rb+3] = dc;
        S_aref[rb] = -B*(vn+v1)-kp; S_aref[rb+1] = -B*(vn-v1)-kp; S_aref[rb+2] = -B*(vn+v2)-kp; S_aref[rb+3] = -B*(vn-v2)-kp; } } }
  WI_(nefc) = rowbase;
  __syncwarp();
}

// ------------------------------------------------------------------ dense Cholesky (packed lower triangle, in place) + solve in shared memory
#define TRI(i, j) ((i)*((i)+1)/2 + (j))
// t -> (i >= j) with t = i(i+1)/2 + j
__device__ __forceinline__ void tri_index(int t, int& i, int& j) {
  i = __float2int_rd((sqrtf(8.0f*t + 1.0f) - 1.0f)*0.5f); if (((i+1)*(i+2) >> 1) <= t) i++; if (((i*(i+1)) >> 1) > t) i--;
  j = t - ((i*(i+1)) >> 1); }

// row-per-lane variant (any n): the n > 36 fallback
__device__ void chol_factor_rows(double* H, int n, int lane) {
  SHARED_PTR(H);
  for (int k = 0; k < n; k++) {
    double dkk = sqrt(fmax(H[TRI(k,k)], MYO_MINVAL));
    __syncwarp();
    if (lane == 0) H[TRI(k,k)] = dkk;
    double inv = 1.0/dkk;
    for (int i = k+1+lane; i < n; i += 32) H[TRI(i,k)] *= inv;
    __syncwarp();
    for (int i = k+1+lane; i < n; i += 32) { double lik = H[TRI(i,k)]; for (int j = k+1; j <= i; j++) H[TRI(i,j)] -= lik*H[TRI(j,k)]; }
    __syncwarp(); }
}
// x <- H^-1 x  (H holds the Cholesky factor)
__device__ void chol_solve(const double* H, int n, double* x, int lane) {
  SHARED_PTR(H); SHARED_PTR(x);
  for (int k = 0; k < n; k++) { double xk = x[k]/H[TRI(k,k)]; __syncwarp(); if (lane == 0) x[k] = xk;
    for (int i = k+1+lane; i < n; i += 32) x[i] -= H[TRI(i,k)]*xk; __syncwarp(); }
  for (int k = n-1; k >= 0; k--) { double xk = x[k]/H[TRI(k,k)]; __syncwarp(); if (lane == 0) x[k] = xk;
    for (int i = lane; i < k; i += 32) x[i] -= H[TRI(k,i)]*xk; __syncwarp(); }
}
// Dense SPD solve for n <= NMAX <= 32, "row in registers, column through shared memory" (root-free L D L'):
// lane i keeps row i of the working lower triangle in registers.  At step k every lane i >= k publishes its (unscaled) entry of
// column k into the packed matrix in shared memory, IN PLACE; after one __syncwarp all lanes read the pivot and the column with
// broadcast LDS (one LDS + one DFMA per trailing entry; round 1's shuffle version spent 2 SHFL + select + DFMA there and needed a
// second register array for the captured columns).  The forward substitution rides along as one more broadcast value per step;
// the backward one reads column `lane` of the stored factor (conflict-free) and broadcasts x_k with one shuffle pair.
// H: packed lower triangle PADDED to NMAX rows (identity rows beyond n; see load_M_dense), destroyed.  x: rhs in / solution out, NMAX slots.
template <int NMAX>
__device__ __noinline__ void chol_rs(double* H, double* x, int n, int lane) {
  SHARED_PTR(H); SHARED_PTR(x);
  const bool own = lane < NMAX; const int rowadr = own ? TRI(lane, 0) : 0;
  double r[NMAX];
  #pragma unroll
  for (int j = 0; j < NMAX; j++) r[j] = (own && j <= lane) ? H[rowadr + j] : 0.0;
  double b = lane < n ? x[lane] : 0.0, invd_own = 1.0;
  __syncwarp();
  #pragma unroll
  for (int k = 0; k < NMAX; k++) {
    if (own && lane >= k) H[rowadr + k] = r[k];      // column k, unscaled (U[i][k] = L[i][k] d_k); lane k: the pivot d_k
    if (lane == k) x[k] = b;                         // z_k of the forward substitution is final (x has chol_pad(n) slots)
    __syncwarp();
    // all broadcast loads of this step are issued as ONE batch, ahead of the reciprocal's dependent chain (left to itself ptxas
    // alternates LDS / DFMA through a single register: one shared-memory latency per trailing entry)
    double col[NMAX];
    #pragma unroll
    for (int j = k+1; j < NMAX; j++) col[j] = H[TRI(j,k)];
    const double dk = H[TRI(k,k)], zk = x[k];
    asm volatile("" ::: "memory");
    const double invd = m_rcp(fmax(dk, MYO_MINVAL));
    if (lane == k) invd_own = invd;
    const double t = r[k]*invd;                      // L[lane][k] on lanes > k
    b = lane > k ? fma(-t, zk, b) : b;
    #pragma unroll
    for (int j = k+1; j < NMAX; j++) r[j] = fma(-t, col[j], r[j]);
  }
  // backward substitution: u_i = z_i - sum_{k>i} U[k][i] x_k ; x_i = u_i / d_i
  #pragma unroll
  for (int k = NMAX-1; k >= 0; k--) { const double xk = __shfl_sync(FULL, b*invd_own, k), hk = (own && lane < k) ? H[TRI(k,0) + lane] : 0.0; b = fma(-hk, xk, b); }
  __syncwarp();
  if (lane < n) x[lane] = b*invd_own;
  __syncwarp();
}

// Bordered root-free L D L' for 32 < n <= 32+E (the legs model: n = 34): H = [A B'; B C] with A the leading 32 x 32 block.  A is eliminated
// exactly like chol_rs<32> (row per lane in registers, columns published in shared memory, batched broadcast loads); the e = n - 32 border
// rows ride along DISTRIBUTED over the lanes (lane j keeps B[q][j]): at step k lane k publishes its now final entries, every lane j > k
// applies the same rank-1 update to its border entries with its own U[j][k].  The e x e Schur complement C - L21 D L21' and the border
// right-hand side are warp sums; the small system is solved redundantly by every lane.  Chosen over a shuffle-based bordered Cholesky,
// which needed two 32-double register arrays (800 spill instructions).
template <int E>
__device__ __noinline__ void chol_rs32b(double* H, double* x, int n, int lane) {
  SHARED_PTR(H); SHARED_PTR(x);
  const int rowadr = TRI(lane, 0);      // n == 32 + E exactly: every border loop is static (a run-time border size cost 8 branches per step: 18.8 k -> see tools/ubench/ubench_chol34.cu)
  double r[32], bq[E];
  #pragma unroll
  for (int j = 0; j < 32; j++) r[j] = j <= lane ? H[rowadr + j] : 0.0;
  #pragma unroll
  for (int q = 0; q < E; q++) bq[q] = H[TRI(32+q, lane)];
  double b = x[lane], invd_own = 1.0;
  __syncwarp();
  #pragma unroll
  for (int k = 0; k < 32; k++) {
    if (lane >= k) H[rowadr + k] = r[k];
    if (lane == k) { x[k] = b;
      #pragma unroll
      for (int q = 0; q < E; q++) H[TRI(32+q, k)] = bq[q]; }
    __syncwarp();
    // the trailing columns are loaded in at most two batches of CH: with 64 row registers, a full batch of 31 and the border values
    // the function overflowed its register budget (196 LDL / 169 STL in SASS)
    constexpr int CH = 18;
    double col[32], bk[E];
    #pragma unroll
    for (int j = k+1; j < 32 && j < k+1+CH; j++) col[j] = H[TRI(j,k)];
    #pragma unroll
    for (int q = 0; q < E; q++) bk[q] = H[TRI(32+q, k)];
    const double dk = H[TRI(k,k)], zk = x[k];
    asm volatile("" ::: "memory");
    const double invd = m_rcp(fmax(dk, MYO_MINVAL));
    if (lane == k) invd_own = invd;
    const double t = r[k]*invd;
    b = lane > k ? fma(-t, zk, b) : b;
    #pragma unroll
    for (int j = k+1; j < 32 && j < k+1+CH; j++) r[j] = fma(-t, col[j], r[j]);
    #pragma unroll
    for (int q = 0; q < E; q++) bq[q] = lane > k ? fma(-bk[q]*invd, r[k], bq[q]) : bq[q];
    if (k+1+CH < 32) {
      #pragma unroll
      for (int j = k+1+CH; j < 32; j++) col[j] = H[TRI(j,k)];
      asm volatile("" ::: "memory");
      #pragma unroll
      for (int j = k+1+CH; j < 32; j++) r[j] = fma(-t, col[j], r[j]); }
  }
  // lane j now holds z1[j] (b), 1/d_j and U[32+q][j] = L21[q][j] d_j (bq).  Schur complement and border right-hand side:
  double S[E][E], y2[E];
  #pragma unroll
  for (int q = 0; q < E; q++) {
    #pragma unroll
    for (int p = 0; p <= q; p++) { const double v = warp_sum(bq[q]*bq[p]*invd_own); S[q][p] = H[TRI(32+q, 32+p)] - v; }
    y2[q] = x[32+q] - warp_sum(bq[q]*invd_own*b); }
  // S = Ls Ds Ls' (root-free, every lane redundantly), x2 = S^-1 y2
  double sinv[E];
  #pragma unroll
  for (int k = 0; k < E; k++) { sinv[k] = m_rcp(fmax(S[k][k], MYO_MINVAL));
    #pragma unroll
    for (int i = k+1; i < E; i++) {
      #pragma unroll
      for (int j = k+1; j <= i; j++) S[i][j] -= S[i][k]*sinv[k]*S[j][k]; }      // (column k still unscaled here)
    #pragma unroll
    for (int i = k+1; i < E; i++) { S[i][k] *= sinv[k]; y2[i] -= S[i][k]*y2[k]; } }
  #pragma unroll
  for (int k = E-1; k >= 0; k--) { y2[k] *= sinv[k];
    #pragma unroll
    for (int i = k+1; i < E; i++) y2[k] -= S[i][k]*y2[i]; }
  // x1 = L^-T D^-1 (z1 - D L21' x2)
  #pragma unroll
  for (int q = 0; q < E; q++) b = fma(-bq[q], y2[q], b);
  #pragma unroll
  for (int k = 31; k >= 0; k--) { const double xk = __shfl_sync(FULL, b*invd_own, k), hk = lane < k ? H[TRI(k,0) + lane] : 0.0; b = fma(-hk, xk, b); }
  __syncwarp();
  x[lane] = b*invd_own;
  #pragma unroll
  for (int q = 0; q < E; q++) if (lane == q) x[32+q] = y2[q];
  __syncwarp();
}

// padded order of the dense solver for an n x n system (the order of the chol_rs instance that solves it; H and the solver vectors are laid out for it)
__host__ __device__ __forceinline__ constexpr int chol_pad(int n) { return n > 32 ? n : (n <= 8 ? 8 : (n == 23 || n == 29 ? n : (n + 3) & ~3)); }
// x <- H^-1 x for a dense SPD H (packed lower triangle in shared memory); H is destroyed
__device__ __forceinline__ void chol_dense(double* H, int n, double* x, int lane) {
  if (n > 36) { chol_factor_rows(H, n, lane); chol_solve(H, n, x, lane); return; }
  if (n > 32) { switch (n) { case 33: chol_rs32b<1>(H, x, n, lane); break; case 34: chol_rs32b<2>(H, x, n, lane); break; case 35: chol_rs32b<3>(H, x, n, lane); break; default: chol_rs32b<4>(H, x, n, lane); break; } return; }
  switch (chol_pad(n)) {
    case 8: chol_rs<8>(H, x, n, lane); break;   case 12: chol_rs<12>(H, x, n, lane); break; case 16: chol_rs<16>(H, x, n, lane); break;
    case 20: chol_rs<20>(H, x, n, lane); break; case 24: chol_rs<24>(H, x, n, lane); break; case 28: chol_rs<28>(H, x, n, lane); break;
    case 23: chol_rs<23>(H, x, n, lane); break; case 29: chol_rs<29>(H, x, n, lane); break; default: chol_rs<32>(H, x, n, lane); break; }
}

// H <- M (+ diag_scale * damping on the diagonal), dense packed lower triangle padded with identity rows up to chol_pad(nv)
template <class MD> __device__ __forceinline__ void load_M_dense(const MD& m, const Warp w, double* H, double diag_scale /* h */) {
  const int n = m.nv, np = chol_pad(n), nt = n*(n+1)/2; for (int i = w.lane; i < np*(np+1)/2; i += 32) H[i] = 0; __syncwarp();
  if (w.lane >= n && w.lane < np) H[TRI(w.lane, w.lane)] = 1.0;
  for (int i = 32 + w.lane; i < np; i += 32) if (i >= n) H[TRI(i, i)] = 1.0;
  (void)nt;
  const idx_t* mi = CI(PM_i); const idx_t* mj = CI(PM_j); const double* dofp = CD(PDOF_d);
  for (int e = w.lane; e < m.nM; e += 32) { int i = mi[e], j = mj[e]; double v = W_(qM)[e]; if (i == j) v += diag_scale*dofp[2*i+1]; H[TRI(i,j)] = v; }
  __syncwarp(); }

// ------------------------------------------------------------------ tree-sparse L'DL (level-scheduled, left-looking) on the qM layout
// Hs (nM, input) -> LD (nM: D on the diagonal slots, unit-L off-diagonals), Dinv (nv)
template <class MD> __device__ void ldl_factor(const MD& m, const Warp w, const double* Hs, double* LD, double* Dinv) {
  SHARED_PTR(Hs); SHARED_PTR(LD); SHARED_PTR(Dinv);
  const idx_t* fadr = CI(PFE_adr); const idx_t* fe = CI(PFE); const idx_t* tadr = CI(PFT_adr); const idx_t* ft = CI(PFT);
  const idx_t* mi = CI(PM_i); const idx_t* mj = CI(PM_j); const idx_t* madr = CI(dof_Madr);
  for (int lev = m.ndepth-1; lev >= 0; lev--) {
    for (int t = fadr[lev] + w.lane; t < fadr[lev+1]; t += 32) { int e = fe[t]; double v = Hs[e];
      for (int q = tadr[t]; q < tadr[t+1]; q++) v -= LD[ft[3*q]]*LD[ft[3*q+1]]*LD[madr[ft[3*q+2]]];
      LD[e] = v; }
    __syncwarp();
    for (int t = fadr[lev] + w.lane; t < fadr[lev+1]; t += 32) { int e = fe[t], k = mi[e];
      if (k == mj[e]) Dinv[k] = 1.0/LD[e]; else LD[e] /= LD[madr[k]]; }
    __syncwarp(); }
}
// x <- (L'DL)^-1 x
template <class MD> __device__ void ldl_solve(const MD& m, const Warp w, const double* LD, const double* Dinv, double* x) {
  SHARED_PTR(LD); SHARED_PTR(Dinv); SHARED_PTR(x);
  const idx_t* ladr = CI(PLV_adr); const idx_t* lv = CI(PLV); const idx_t* dadr = CI(PDS_adr); const idx_t* ds = CI(PDS);
  const idx_t* madr = CI(dof_Madr); const idx_t* mj = CI(PM_j);
  for (int lev = m.ndepth-1; lev >= 0; lev--) {
    for (int t = ladr[lev] + w.lane; t < ladr[lev+1]; t += 32) { int j = lv[t]; double s = x[j];
      for (int q = dadr[j]; q < dadr[j+1]; q++) s -= LD[ds[2*q+1]]*x[ds[2*q]];
      x[j] = s; }
    __syncwarp(); }
  for (int lev = 0; lev < m.ndepth; lev++) {
    for (int t = ladr[lev] + w.lane; t < ladr[lev+1]; t += 32) { int i = lv[t]; double s = x[i]*Dinv[i];
      for (int e = madr[i]+1; e <= madr[i]+lev; e++) s -= LD[e]*x[mj[e]];
      x[i] = s; }
    __syncwarp(); }
}

// ------------------------------------------------------------------ Newton solver: leaves qacc in S_a
// Called by EVERY warp of the CTA when cta_sync is set (live = this warp holds an env): the warps still iterating are re-aligned by CTA
// barriers at the top of each Newton iteration and before the Cholesky, so that they keep sharing instruction fetches inside the
// phase too (a lone register Cholesky out of step with the other warps fetches its code alone); finished and idle
// warps only take part in the barriers.  The total wait is unchanged: the CTA leaves the phase with its slowest env either way.
// __forceinline__: as a real call the function receives the DevModel by address and every m.field becomes a generic load that is repeated
// after each shared-memory store (measured round 2: 310 LD.E in the solver of the launch_bounds(448) kernel, which had not inlined it).
template <class MD> __device__ __forceinline__ void phase_solve(const MD& m, const Warp w, double tol, long long* cyc, bool live, bool cta_sync) {
  long long tc = cyc ? clock64() : 0;
  #define LAP(k) if (cyc) { long long t_ = clock64(); cyc[k] += t_ - tc; tc = t_; }
  int n = m.nv, nefc = live ? WI_(nefc) : 0; const int ncon = live ? WI_(ncon) : 0, nlimrow = live ? WI_(nlimrow) : 0; int niter = 0;
  bool active = live;
  if (live && nefc == 0) {   // unconstrained: qacc = M^-1 qfrc_smooth
    ldl_factor(m, w, W_(qM), S_LD, S_Dinv);
    for (int i = w.lane; i < n; i += 32) { S_a[i] = W_(fsm)[i]; S_Ma[i] = W_(fsm)[i]; } __syncwarp();
    ldl_solve(m, w, S_LD, S_Dinv, S_a); active = false; }
  if (active) {
    for (int i = w.lane; i < n; i += 32) S_a[i] = W_(qws)[i]; __syncwarp();
    mul_M(m, w, S_Ma, S_a); rows_apply(m, w, S_a, S_jar); __syncwarp();
    for (int r = w.lane; r < nefc; r += 32) S_jar[r] -= S_aref[r]; __syncwarp(); }
  const double scale = 1.0/(m.meaninertia*(n > 1 ? n : 1));
  const idx_t* eq = CI(PEQ); const idx_t* pr = CI(PPAIR); const idx_t* path = CI(PPATH);
  for (int iter = 0; iter < 50; iter++) {
    if (cta_sync) { if (!__syncthreads_or(active ? 1 : 0)) break; } else if (!active) break;
    bool dense = false;
    if (active) {
    // gradient
    for (int i = w.lane; i < n; i += 32) S_g[i] = S_Ma[i]-W_(fsm)[i];
    for (int r = w.lane; r < nefc; r += 32) { double x = S_jar[r]; S_jv[r] = (r < m.neq || x < 0) ? S_D[S_drow[r]]*x : 0.0; }   // jv used as scratch weights
    __syncwarp(); rows_applyT_add(m, w, S_jv, S_g); __syncwarp();
    double gn = 0; for (int i = w.lane; i < n; i += 32) gn += S_g[i]*S_g[i]; gn = sqrt(warp_sum(gn));
    LAP(8)
    if (scale*gn < tol) active = false; }
    if (active) {
    if (cyc) cyc[14]++;
    // Hessian: tree-sparse L'DL when no contact row is active (limits/equalities keep M's sparsity), dense Cholesky otherwise
    dense = (m.neq > 0 && !m.eq_tree);
    for (int c = w.lane; c < ncon && !dense; c += 32) { const int rn = S_crown[c], nr = CNR(rn), rb = CROW(rn); for (int r = 0; r < nr; r++) if (S_jar[rb+r] < 0) dense = true; }
    dense = __any_sync(FULL, dense);
    for (int i = w.lane; i < n; i += 32) S_p[i] = -S_g[i];      // (p shares g's storage: the gradient is not read again this iteration)
    __syncwarp();
    if (cyc && dense) cyc[15]++;
    if (!dense) {
      const idx_t* madr = CI(dof_Madr);
      for (int e = w.lane; e < m.nM; e += 32) S_Hs[e] = W_(qM)[e];
      __syncwarp();
      if (w.lane == 0) for (int e = 0; e < m.neq; e++) { int d1 = eq[PEQ_ISTRIDE*e+1], d2 = eq[PEQ_ISTRIDE*e+3]; double De = S_D[e], j2 = S_eqJ[e]; S_Hs[madr[d1]] += De;
        if (d2 >= 0) { S_Hs[eq[PEQ_ISTRIDE*e+4]] += De*j2; S_Hs[madr[d2]] += De*j2*j2; } }
      __syncwarp();
      for (int pass = 0; pass < 2; pass++) { for (int r = w.lane; r < nlimrow; r += 32) { int dsc = S_lrow[r]; if (((dsc >> 8) & 1) == pass && S_jar[m.neq+r] < 0) S_Hs[madr[dsc & 0xff]] += S_D[m.neq+r]; } __syncwarp(); }
      LAP(9)
      ldl_factor(m, w, S_Hs, S_LD, S_Dinv); ldl_solve(m, w, S_LD, S_Dinv, S_p);
      LAP(10)
    } else {
    load_M_dense(m, w, S_H, 0.0);
    if (w.lane == 0) for (int e = 0; e < m.neq; e++) { int d1 = eq[PEQ_ISTRIDE*e+1], d2 = eq[PEQ_ISTRIDE*e+3]; double De = S_D[e], j2 = S_eqJ[e]; S_H[TRI(d1,d1)] += De;
      if (d2 >= 0) { S_H[d1 > d2 ? TRI(d1,d2) : TRI(d2,d1)] += De*j2; S_H[TRI(d2,d2)] += De*j2*j2; } }
    __syncwarp();
    for (int pass = 0; pass < 2; pass++) { for (int r = w.lane; r < nlimrow; r += 32) { int dsc = S_lrow[r]; if (((dsc >> 8) & 1) == pass && S_jar[m.neq+r] < 0) { int d = dsc & 0xff; S_H[TRI(d,d)] += S_D[m.neq+r]; } } __syncwarp(); }
    // contacts: J' W J, one contact at a time, the lanes over the lower triangle of its block.  (The gather form that pays for the
    // gradient does not pay here: with one H entry per lane nearly every contact hits SOME lane and the warp runs the hit path 9 x ncon times.)
    for (int c = 0; c < ncon; c++) { const int rn = S_crown[c], nr = CNR(rn), rb = CROW(rn); if (!nr) continue; const idx_t* q = pr + PPAIR_ISTRIDE*S_cpair[c]; double W[6] = {0,0,0,0,0,0};  // nn n1 n2 11 12 22
      if (nr == 1) { if (S_jar[rb] < 0) W[0] = S_D[S_DCON(c)]; }
      else { const double Dv = S_D[S_DCON(c)];
        double a0 = S_jar[rb] < 0 ? Dv : 0, a1 = S_jar[rb+1] < 0 ? Dv : 0, a2 = S_jar[rb+2] < 0 ? Dv : 0, a3 = S_jar[rb+3] < 0 ? Dv : 0;
        W[0] = a0+a1+a2+a3; W[1] = a0-a1; W[2] = a2-a3; W[3] = a0+a1; W[5] = a2+a3; }
      if (W[0] != 0) { const JacRef J = S_jac(c); int np = q[4], ntri = (np*(np+1)) >> 1;
        for (int t = w.lane; t < ntri; t += 32) { int ei, ej;
          if (np <= 8) { ei = (t >= 1) + (t >= 3) + (t >= 6) + (t >= 10) + (t >= 15) + (t >= 21) + (t >= 28); ej = t - ((ei*(ei+1)) >> 1); } else tri_index(t, ei, ej);
          const JacRef ja = J + 3*ei, jb = J + 3*ej; const double a[3] = {ja[0], ja[1], ja[2]}, b[3] = {jb[0], jb[1], jb[2]};
          double wa0 = W[0]*a[0]+W[1]*a[1]+W[2]*a[2], wa1 = W[1]*a[0]+W[3]*a[1], wa2 = W[2]*a[0]+W[5]*a[2];
          int di = path[q[3]+ei] >> 1, dj = path[q[3]+ej] >> 1; S_H[TRI(di,dj)] += wa0*b[0]+wa1*b[1]+wa2*b[2]; } }
      __syncwarp(); }
    LAP(9)
    } }
    if (cta_sync) __syncthreads();
    if (active) {
    if (dense) { chol_dense(S_H, n, S_p, w.lane); LAP(10) }
    // exact line search along p
    mul_M(m, w, S_Mp, S_p); rows_apply(m, w, S_p, S_jv); __syncwarp();
    double ga = 0, gb = 0; for (int i = w.lane; i < n; i += 32) { ga += S_p[i]*(S_Ma[i]-W_(fsm)[i]); gb += S_p[i]*S_Mp[i]; } ga = warp_sum(ga); gb = warp_sum(gb);
    double alpha = 0, lo = 0, hi = -1, d0 = 0;
    for (int it = 0; it < 40; it++) { double dv = 0, hh = 0;
      for (int r = w.lane; r < nefc; r += 32) { double x = S_jar[r]+alpha*S_jv[r]; if (r < m.neq || x < 0) { const double Dr = S_D[S_drow[r]], jv = S_jv[r]; dv += Dr*x*jv; hh += Dr*jv*jv; } }
      dv = warp_sum(dv) + ga + gb*alpha; hh = warp_sum(hh) + gb;
      if (it == 0) { d0 = fabs(dv); if (dv >= 0) break; } else { if (dv < 0) lo = alpha; else hi = alpha; if (fabs(dv) <= 1e-10*d0) break; }
      double an = alpha - dv*m_rcp(hh);
      if (it > 0 && (an <= lo || (hi > 0 && an >= hi))) an = hi > 0 ? 0.5*(lo+hi) : 2*alpha+1;
      if (an == alpha) break;
      alpha = an; }
    if (alpha == 0) active = false;   // no descent possible: converged to round-off
    else {
    for (int i = w.lane; i < n; i += 32) { S_a[i] += alpha*S_p[i]; S_Ma[i] += alpha*S_Mp[i]; }
    // rows that switch between active and inactive along the step; with none the cost was exactly quadratic along p, the Newton
    // step (alpha = 1) lands on its minimum and the gradient vanishes to round-off: converged without another gradient pass
    bool flip = false;
    for (int r = w.lane; r < nefc; r += 32) { double x0 = S_jar[r], x1 = x0 + alpha*S_jv[r]; S_jar[r] = x1; if (r >= m.neq && (x0 < 0) != (x1 < 0)) flip = true; }
    __syncwarp(); niter = iter+1; LAP(11)
    if (!__any_sync(FULL, flip)) active = false; } } }
  if (live) WI_(niter) = niter;
  #undef LAP
}

// ------------------------------------------------------------------ semi-implicit Euler with implicit joint damping
// qpos <- qpos (+) h v (mj_integratePos): hinge and slide joints add; a free joint adds the position and turns its quaternion by
// exp(h omega / 2) in the body frame, then normalises it.  Lanes over the joints; the caller syncs.  phase_integrate keeps its own
// inline copy of this loop over qpos / qvel, for the same reason as phase_constraints' equality rows.
template <class MD> __device__ __forceinline__ void integrate_pos(const MD& m, const Warp w, double* qpos, const double* v, double h) {
  const idx_t* jtype = CI(jnt_type); const idx_t* jq = CI(jnt_qposadr); const idx_t* jd = CI(jnt_dofadr);
  for (int j = w.lane; j < m.njnt; j += 32) { int qa = jq[j], da = jd[j];
    if (jtype[j] == 0) { for (int c = 0; c < 3; c++) qpos[qa+c] += h*v[da+c];
      double wv[3] = {v[da+3], v[da+4], v[da+5]}, nn = sqrt(dot3(wv,wv)), ang = h*nn;
      if (nn < MYO_MINVAL) { wv[0]=1; wv[1]=0; wv[2]=0; } else { wv[0]/=nn; wv[1]/=nn; wv[2]/=nn; }
      double sn, cs; sincos(0.5*ang, &sn, &cs); double ql[4] = {cs, wv[0]*sn, wv[1]*sn, wv[2]*sn}, qn[4]; quat_mul(qn, qpos+qa+3, ql); quat_norm(qn);
      for (int c = 0; c < 4; c++) qpos[qa+3+c] = qn[c]; }
    else qpos[qa] += h*v[da]; }
}

// v <- q2 (-) q1 (mj_differentiatePos with dt = 1): hinge and slide joints and a free joint's position subtract; a free joint's quaternion
// gives mju_subQuat(q2, q1), the rotation vector of q1^-1 q2 in the body frame (the frame integrate_pos turns in), angle in (-pi, pi].
// The vector part of q1^-1 q2 is formed without fused multiply-adds, so that equal quaternions give exactly 0 (a contracted
// a0 b1 - b0 a1 leaves the rounding error of one product, which divided by eps would put ~1e-11 into columns that are exactly 0).
// Lanes over the joints; the caller syncs.
template <class MD> __device__ __forceinline__ void differentiate_pos(const MD& m, const Warp w, double* v, const double* q1, const double* q2) {
  const idx_t* jtype = CI(jnt_type); const idx_t* jq = CI(jnt_qposadr); const idx_t* jd = CI(jnt_dofadr);
  for (int j = w.lane; j < m.njnt; j += 32) { int qa = jq[j], da = jd[j];
    if (jtype[j] == 0) { for (int c = 0; c < 3; c++) v[da+c] = q2[qa+c] - q1[qa+c];
      const double* a = q1 + qa + 3; const double* b = q2 + qa + 3;
      #define M_(x, y) __dmul_rn(x, y)
      const double d[4] = {__dadd_rn(__dadd_rn(__dadd_rn(M_(a[0], b[0]), M_(a[1], b[1])), M_(a[2], b[2])), M_(a[3], b[3])),      // conj(a) b
        __dsub_rn(__dsub_rn(M_(a[0], b[1]), M_(b[0], a[1])), __dsub_rn(M_(a[2], b[3]), M_(a[3], b[2]))),
        __dsub_rn(__dsub_rn(M_(a[0], b[2]), M_(b[0], a[2])), __dsub_rn(M_(a[3], b[1]), M_(a[1], b[3]))),
        __dsub_rn(__dsub_rn(M_(a[0], b[3]), M_(b[0], a[3])), __dsub_rn(M_(a[1], b[2]), M_(a[2], b[1])))};
      #undef M_
      double ax[3] = {d[1], d[2], d[3]}; const double s = sqrt(dot3(ax, ax));
      if (s < MYO_MINVAL) { ax[0] = 1; ax[1] = 0; ax[2] = 0; } else { const double r = 1.0/s; ax[0] *= r; ax[1] *= r; ax[2] *= r; }
      const double PI = 3.14159265358979323846; double ang = 2*atan2(s, d[0]); if (ang > PI) ang -= 2*PI;
      for (int c = 0; c < 3; c++) v[da+3+c] = ax[c]*ang; }
    else v[da] = q2[qa] - q1[qa]; }
}

template <class MD> __device__ void phase_integrate(const MD& m, const Warp w, long long* cyc) {
  int n = m.nv; double h = m.timestep; long long tc = cyc ? clock64() : 0;
  // (M + h B) qacc' = M qacc  (= qfrc_smooth + qfrc_constraint at the solver optimum)
  for (int i = w.lane; i < n; i += 32) S_g[i] = S_Ma[i];     // M qacc, maintained by the solver
  __syncwarp();
  if (n >= 8 && n <= 36) {     // mid-size systems: the register Cholesky beats the level-scheduled sparse factorisation (long index-chasing chains)
    load_M_dense(m, w, S_H, h);
    if (cyc) { long long t_ = clock64(); cyc[18] += t_ - tc; tc = t_; }
    chol_dense(S_H, n, S_g, w.lane);
  } else {
  { const idx_t* mi = CI(PM_i); const idx_t* mj = CI(PM_j); const double* dofp = CD(PDOF_d);
    for (int e = w.lane; e < m.nM; e += 32) { double v = W_(qM)[e]; if (mi[e] == mj[e]) v += h*dofp[2*mi[e]+1]; S_Hs[e] = v; } __syncwarp(); }
  if (cyc) { long long t_ = clock64(); cyc[18] += t_ - tc; tc = t_; }
  ldl_factor(m, w, S_Hs, S_LD, S_Dinv); ldl_solve(m, w, S_LD, S_Dinv, S_g);
  }
  if (cyc) { long long t_ = clock64(); cyc[19] += t_ - tc; tc = t_; }
  for (int i = w.lane; i < n; i += 32) { W_(qvel)[i] += h*S_g[i]; W_(qws)[i] = S_a[i]; }
  __syncwarp();
  const idx_t* jtype = CI(jnt_type); const idx_t* jq = CI(jnt_qposadr); const idx_t* jd = CI(jnt_dofadr);
  for (int j = w.lane; j < m.njnt; j += 32) { int qa = jq[j], da = jd[j];
    if (jtype[j] == 0) { for (int c = 0; c < 3; c++) W_(qpos)[qa+c] += h*W_(qvel)[da+c];
      double wv[3] = {W_(qvel)[da+3], W_(qvel)[da+4], W_(qvel)[da+5]}, nn = sqrt(dot3(wv,wv)), ang = h*nn;
      if (nn < MYO_MINVAL) { wv[0]=1; wv[1]=0; wv[2]=0; } else { wv[0]/=nn; wv[1]/=nn; wv[2]/=nn; }
      double sn, cs; sincos(0.5*ang, &sn, &cs); double ql[4] = {cs, wv[0]*sn, wv[1]*sn, wv[2]*sn}, qn[4]; quat_mul(qn, W_(qpos)+qa+3, ql); quat_norm(qn);
      for (int c = 0; c < 4; c++) W_(qpos)[qa+3+c] = qn[c]; }
    else W_(qpos)[qa] += h*W_(qvel)[da]; }
  __syncwarp();
}
