/* ik_oracle.c -- mj_jacSite and damped least-squares inverse kinematics on the CPU oracle (test infrastructure only; compiled by
 * tests/ik_oracle.py).
 *
 * The oracle's own source is included unchanged.  What this file adds:
 *   oracle_jac_site   MuJoCo's mj_jacSite: the oracle's kinematics (quaternion chain) and com_pos (cdof about the subtree centre of
 *                     mass), then jac_point at the site, so that the device's dof axes and anchors are set against MuJoCo's cdof route
 *   oracle_ik         the semantics of myo_batch_ik (include/myo_b200.h) restated step by step on dense nv x nv matrices: the site
 *                     Jacobians from jac_point, the joint equalities from the model's eq_data (not the kernel program's tables), a
 *                     Cholesky solve, mj_integratePos and the range clamp */
#include "../oracle/myo_oracle.c"

/* site pose at the oracle's current kinematics: position, rotation matrix and quaternion (xquat of the body times site_quat) */
static void site_pose(ora* o, int sid, const double* squat, double* pos, double* mat, double* quat) {
  const int b = ISEC(o,site_bodyid)[sid]; const double* sp = DSEC(o,site_pos) + 3*sid; double v[3];
  mat_vec(v, o->xmat+9*b, sp); for (int k=0;k<3;k++) pos[k]=o->xpos[3*b+k]+v[k];
  quat_mul(quat, o->xquat+4*b, squat); quat_norm(quat); quat2mat(mat, quat);
}

/* mj_jacSite at the oracle's qpos: jacp, jacr [3, nv] (nullable), site position and rotation */
void oracle_jac_site(ora* o, int sid, const double* squat, double* jacp, double* jacr, double* pos, double* mat) {
  double q[4]; kinematics(o); com_pos(o); site_pose(o, sid, squat, pos, mat, q);
  jac_point(o, jacp, jacr, pos, ISEC(o,site_bodyid)[sid]);
}

/* dm_control's quat2vel(target * conj(site_xquat)): rotation vector, angle in [0, pi] */
static void quat_err(const double* target, const double* q, double* out) {
  double c[4] = {q[0], -q[1], -q[2], -q[3]}, e[4]; quat_mul(e, target, c);
  if (e[0] < 0) for (int k=0;k<4;k++) e[k] = -e[k];
  double sn = sqrt(e[1]*e[1]+e[2]*e[2]+e[3]*e[3]);
  if (sn == 0) { out[0]=out[1]=out[2]=0; return; }
  double ang = 2*atan2(sn, e[0]); for (int k=0;k<3;k++) out[k] = e[1+k]/sn*ang;
}

/* q <- q (+) dq: mj_integratePos with dt = 1 (free joints: position added, quaternion times exp(omega / 2) in the body frame, normalised) */
static void integrate_pos_ref(ora* o, const double* dq) {
  const int *jtype=ISEC(o,jnt_type), *jq=ISEC(o,jnt_qposadr), *jd=ISEC(o,jnt_dofadr);
  for (int j=0;j<o->njnt;j++) { double* q=o->qpos+jq[j]; const double* v=dq+jd[j];
    if (jtype[j]==JNT_FREE) { for (int k=0;k<3;k++) q[k]+=v[k];
      double ax[3]={v[3],v[4],v[5]}, ang=normalize3(ax), ql[4], qn[4]; axisangle_quat(ql, ax, ang); quat_mul(qn, q+3, ql); quat_norm(qn); memcpy(q+3, qn, 32); }
    else q[0]+=v[0]; }
}

/* inverse kinematics from the oracle's qpos (left there); outputs nullable.  squat [ns, 4]; weight [ns, 2] nullable; tquat [ns, 4]
 * nullable; qref [nq] nullable (the start); mask [nv] nullable */
void oracle_ik(ora* o, int ns, const int* sid, const double* squat, const double* weight, const double* tpos, const double* tquat,
               const double* qref_in, const unsigned char* mask, int max_iter, double tol, double damping, double max_step, double rho, double weq,
               int* niter, int* converged, double* err, double* sxpos, double* sxmat, double* jacp, double* jacr) {
  const int nv=o->nv, nq=o->nq;
  const int *jtype=ISEC(o,jnt_type), *jq=ISEC(o,jnt_qposadr), *jd=ISEC(o,jnt_dofadr), *lim=ISEC(o,jnt_limited), *sb=ISEC(o,site_bodyid);
  const int *e1=ISEC(o,eq_obj1id), *e2=ISEC(o,eq_obj2id), *eact=ISEC(o,eq_active0);
  const double *range=DSEC(o,jnt_range), *edata=DSEC(o,eq_data), *qpos0=DSEC(o,qpos0);
  double* qref=dalloc(nq); memcpy(qref, qref_in ? qref_in : o->qpos, sizeof(double)*nq);
  double *P=dalloc(3*ns), *Rm=dalloc(9*ns), *E=dalloc(3*ns), *W=dalloc(3*ns), *ep=dalloc(ns), *er=dalloc(ns);
  double *Jp=dalloc(3*nv), *Jr=dalloc(3*nv), *H=dalloc((size_t)nv*nv), *g=dalloc(nv), *row=dalloc(nv);
  for (int it=0;;it++) {
    /* 1-3: kinematics, residuals, stop test */
    kinematics(o); com_pos(o);
    int ok=1;
    for (int s=0;s<ns;s++) { double q[4]; site_pose(o, sid[s], squat+4*s, P+3*s, Rm+9*s, q);
      for (int k=0;k<3;k++) E[3*s+k]=tpos[3*s+k]-P[3*s+k];
      ep[s]=norm3(E+3*s); er[s]=0; W[3*s]=W[3*s+1]=W[3*s+2]=0;
      if (tquat) { double t[4]; memcpy(t, tquat+4*s, 32); quat_norm(t); quat_err(t, q, W+3*s); er[s]=norm3(W+3*s); }
      if (!(ep[s]<=tol && (!tquat || er[s]<=tol))) ok=0; }
    if (ok || it==max_iter) {
      if (niter) *niter=it;
      if (converged) *converged=ok;
      for (int s=0;s<ns;s++) {
        if (err) { err[2*s]=ep[s]; err[2*s+1]=er[s]; }
        if (sxpos) memcpy(sxpos+3*s, P+3*s, 24);
        if (sxmat) memcpy(sxmat+9*s, Rm+9*s, 72);
        if (jacp || jacr) jac_point(o, jacp ? jacp+(size_t)3*nv*s : NULL, jacr ? jacr+(size_t)3*nv*s : NULL, P+3*s, sb[sid[s]]); }
      break; }
    /* 4-5: Jacobians and the normal equations */
    memset(H, 0, sizeof(double)*nv*nv); memset(g, 0, sizeof(double)*nv);
    for (int s=0;s<ns;s++) { const double wp=weight ? weight[2*s] : 1, wr=weight ? weight[2*s+1] : 1;
      jac_point(o, Jp, Jr, P+3*s, sb[sid[s]]);
      for (int r=0;r<3;r++) for (int i=0;i<nv;i++) { g[i]+=wp*Jp[r*nv+i]*E[3*s+r]; if (tquat) g[i]+=wr*Jr[r*nv+i]*W[3*s+r];
        for (int j=0;j<nv;j++) { H[i*nv+j]+=wp*Jp[r*nv+i]*Jp[r*nv+j]; if (tquat) H[i*nv+j]+=wr*Jr[r*nv+i]*Jr[r*nv+j]; } } }
    for (int e=0;e<o->neq;e++) { if (!eact[e]) continue;      /* joint equalities (every equality of the shipped models) */
      const int j1=e1[e], j2=e2[e]; const double* c=edata+5*e; memset(row, 0, sizeof(double)*nv);
      double res=o->qpos[jq[j1]]-qpos0[jq[j1]]; row[jd[j1]]=1;
      if (j2<0) res-=c[0];
      else { double x=o->qpos[jq[j2]]-qpos0[jq[j2]], poly=c[0]+c[1]*x+c[2]*x*x+c[3]*x*x*x+c[4]*x*x*x*x; res-=poly; row[jd[j2]]=-(c[1]+2*c[2]*x+3*c[3]*x*x+4*c[4]*x*x*x); }
      for (int i=0;i<nv;i++) { g[i]-=weq*row[i]*res; for (int j=0;j<nv;j++) H[i*nv+j]+=weq*row[i]*row[j]; } }
    for (int j=0;j<o->njnt;j++) if (jtype[j]==JNT_HINGE || jtype[j]==JNT_SLIDE) { const int d=jd[j]; H[d*nv+d]+=rho; g[d]+=rho*(qref[jq[j]]-o->qpos[jq[j]]); }
    for (int i=0;i<nv;i++) H[i*nv+i]+=damping;
    /* 6: dof mask */
    if (mask) for (int i=0;i<nv;i++) if (!mask[i]) { for (int j=0;j<nv;j++) H[i*nv+j]=H[j*nv+i]=0; H[i*nv+i]=1; g[i]=0; }
    /* 7: Cholesky solve and step cap */
    for (int k=0;k<nv;k++) { double s=H[k*nv+k]; for (int p=0;p<k;p++) s-=H[k*nv+p]*H[k*nv+p]; s=sqrt(s); H[k*nv+k]=s;
      for (int i=k+1;i<nv;i++) { double t=H[i*nv+k]; for (int p=0;p<k;p++) t-=H[i*nv+p]*H[k*nv+p]; H[i*nv+k]=t/s; } }
    for (int i=0;i<nv;i++) { double t=g[i]; for (int p=0;p<i;p++) t-=H[i*nv+p]*g[p]; g[i]=t/H[i*nv+i]; }
    for (int i=nv-1;i>=0;i--) { double t=g[i]; for (int p=i+1;p<nv;p++) t-=H[p*nv+i]*g[p]; g[i]=t/H[i*nv+i]; }
    double n2=0; for (int i=0;i<nv;i++) n2+=g[i]*g[i];
    if (sqrt(n2)>max_step) { double sc=max_step/sqrt(n2); for (int i=0;i<nv;i++) g[i]*=sc; }
    /* 8: update and range clamp */
    integrate_pos_ref(o, g);
    for (int j=0;j<o->njnt;j++) if (lim[j] && (jtype[j]==JNT_HINGE || jtype[j]==JNT_SLIDE)) o->qpos[jq[j]]=clip(o->qpos[jq[j]], range[2*j], range[2*j+1]);
  }
  free(qref); free(P); free(Rm); free(E); free(W); free(ep); free(er); free(Jp); free(Jr); free(H); free(g); free(row);
}
