/* fd_oracle.c -- MuJoCo's mjd_transitionFD on the CPU oracle (test infrastructure only; compiled by tests/fd_oracle.py).
 *
 * tests/rollout_oracle.c (and through it the oracle's source) is included unchanged.  oracle_transition_fd restates mjd_stepFD on dense
 * arrays, with one mj_step replaced by one interval of `substeps` oracle_step_applied calls with ctrl held:
 *   save the state and warm start; run the nominal interval and one interval per perturbed column from the saved start, each with the
 *   saved warm start and the inverse-wrap roots reset cold (wrap_warm = 1 from wrap_z = -1, the rule of the device's intervals);
 *   perturb qpos column j by integratePos(qpos, e_j, +-eps), qvel / act column j by +-eps, ctrl column i by +-eps where
 *   fwd = !limited || inRange(c, c + eps) and back = (centered || !fwd) && (!limited || inRange(c - eps, c));
 *   difference both sides (x'+ (-) x'-) * (1 / (2 eps)), one side (x'+ (-) x'0) * (1 / eps) or (x'0 (-) x'-) * (1 / eps), neither 0,
 *   where (-) is differentiatePos on qpos and subtraction on qvel and act; then restore the saved state. */
#include "rollout_oracle.c"

/* mj_integratePos: qpos <- qpos (+) scale v (a free joint turns its quaternion in the body frame, then normalises it) */
void oracle_integrate_pos(const ora* o, double* qpos, const double* v, double scale) {
  const int *jtype=ISEC(o,jnt_type), *jq=ISEC(o,jnt_qposadr), *jd=ISEC(o,jnt_dofadr);
  for (int j=0;j<o->njnt;j++) { int qa=jq[j], da=jd[j];
    if (jtype[j]==JNT_FREE) { for (int k=0;k<3;k++) qpos[qa+k]+=scale*v[da+k];
      double w[3]={v[da+3],v[da+4],v[da+5]}, ang=scale*normalize3(w), ql[4], qn[4];
      axisangle_quat(ql,w,ang); quat_mul(qn,qpos+qa+3,ql); quat_norm(qn); memcpy(qpos+qa+3,qn,32); }
    else qpos[qa]+=scale*v[da]; }
}

/* mj_differentiatePos: v <- (q2 (-) q1) / dt; a free joint's quaternion gives mju_subQuat(q2, q1), the rotation vector of q1^-1 q2 */
void oracle_differentiate_pos(const ora* o, double* v, double dt, const double* q1, const double* q2) {
  const int *jtype=ISEC(o,jnt_type), *jq=ISEC(o,jnt_qposadr), *jd=ISEC(o,jnt_dofadr);
  for (int j=0;j<o->njnt;j++) { int qa=jq[j], da=jd[j];
    if (jtype[j]==JNT_FREE) { for (int k=0;k<3;k++) v[da+k]=(q2[qa+k]-q1[qa+k])/dt;
      const double* a=q1+qa+3; double qneg[4]={a[0],-a[1],-a[2],-a[3]}, d[4]; quat_mul(d,qneg,q2+qa+3);
      double ax[3]={d[1],d[2],d[3]}, s=norm3(ax);
      if (s<MINVAL) { ax[0]=1; ax[1]=0; ax[2]=0; } else { double r=1/s; ax[0]*=r; ax[1]*=r; ax[2]*=r; }
      double ang=2*atan2(s,d[0]); if (ang>M_PI) ang-=2*M_PI;
      for (int k=0;k<3;k++) v[da+3+k]=ax[k]*ang/dt; }
    else v[da]=(q2[qa]-q1[qa])/dt; }
}

/* one interval from the start (qpos, qvel, act, warm start) with ctrl held; the result state [qpos | qvel | act] into out */
static void fd_interval(ora* o, const double* q, const double* v, const double* a, const double* w, const double* ctrl, const double* f,
                        int substeps, double* out) {
  int nq=o->nq, nv=o->nv, na=o->na;
  memcpy(o->qpos,q,8*nq); memcpy(o->qvel,v,8*nv); memcpy(o->act,a,8*na); memcpy(o->qacc_warmstart,w,8*nv); memcpy(o->ctrl,ctrl,8*o->nu);
  o->wrap_warm=1; for (int k=0;k<o->nwrap;k++) o->wrap_z[k]=-1;
  for (int s=0;s<substeps;s++) oracle_step_applied(o,f);
  memcpy(out,o->qpos,8*nq); memcpy(out+nq,o->qvel,8*nv); memcpy(out+nq+nv,o->act,8*na);
}

/* mjd_stepFD's clampedStateDiff: column of d x' into ds [nx] from the nominal x0 and the + / - results (either may be NULL) */
static void fd_diff(const ora* o, double* ds, const double* x0, const double* xp, const double* xm, double eps) {
  int nq=o->nq, nv=o->nv, na=o->na, nx=2*nv+na; const double *s1, *s2; double h;
  if (xp && xm) { s1=xm; s2=xp; h=2*eps; } else if (xp) { s1=x0; s2=xp; h=eps; } else if (xm) { s1=xm; s2=x0; h=eps; }
  else { memset(ds,0,8*nx); return; }
  oracle_differentiate_pos(o,ds,1,s1,s2);
  for (int i=0;i<nv+na;i++) ds[nv+i]=s2[nq+i]-s1[nq+i];
  double r=1/h; for (int i=0;i<nx;i++) ds[i]*=r;
}

static int in_range(double x1, double x2, const double* b) { return x1>=b[0] && x1<=b[1] && x2>=b[0] && x2<=b[1]; }

void oracle_transition_fd(ora* o, const double* ctrl, const double* qfrc_applied, double eps, int centered, int substeps, double* A, double* B) {
  int nq=o->nq, nv=o->nv, na=o->na, nu=o->nu, nx=2*nv+na, ns=nq+nv+na;
  double *q0=dalloc(nq), *v0=dalloc(nv), *a0=dalloc(na), *w0=dalloc(nv), t0=o->time, ww0=o->wrap_warm, *wz0=dalloc(o->nwrap);
  memcpy(q0,o->qpos,8*nq); memcpy(v0,o->qvel,8*nv); memcpy(a0,o->act,8*na); memcpy(w0,o->qacc_warmstart,8*nv); memcpy(wz0,o->wrap_z,8*o->nwrap);
  double *f=dalloc(nv), *x0=dalloc(ns), *xp=dalloc(ns), *xm=dalloc(ns), *ds=dalloc(nx), *q=dalloc(nq), *v=dalloc(nv), *a=dalloc(na), *e=dalloc(nv), *c=dalloc(nu);
  if (qfrc_applied) memcpy(f,qfrc_applied,8*nv);
  memcpy(c,ctrl,8*nu);
  fd_interval(o,q0,v0,a0,w0,c,f,substeps,x0);
  if (A) for (int j=0;j<nx;j++) {
    for (int side=0; side<(centered ? 2 : 1); side++) { const double h = side ? -eps : eps;
      memcpy(q,q0,8*nq); memcpy(v,v0,8*nv); memcpy(a,a0,8*na);
      if (j<nv) { memset(e,0,8*nv); e[j]=1; oracle_integrate_pos(o,q,e,h); }
      else if (j<2*nv) v[j-nv]+=h; else a[j-2*nv]+=h;
      fd_interval(o,q,v,a,w0,c,f,substeps,side ? xm : xp); }
    fd_diff(o,ds,x0,xp,centered ? xm : NULL,eps);
    for (int i=0;i<nx;i++) A[(size_t)i*nx+j]=ds[i]; }
  if (B) { const int* lim=ISEC(o,actuator_ctrllimited); const double* cr=DSEC(o,actuator_ctrlrange);
    for (int i=0;i<nu;i++) {
      int fwd = !lim[i] || in_range(ctrl[i],ctrl[i]+eps,cr+2*i);
      if (fwd) { c[i]=ctrl[i]+eps; fd_interval(o,q0,v0,a0,w0,c,f,substeps,xp); c[i]=ctrl[i]; }
      int back = (centered || !fwd) && (!lim[i] || in_range(ctrl[i]-eps,ctrl[i],cr+2*i));
      if (back) { c[i]=ctrl[i]-eps; fd_interval(o,q0,v0,a0,w0,c,f,substeps,xm); c[i]=ctrl[i]; }
      fd_diff(o,ds,x0,fwd ? xp : NULL,back ? xm : NULL,eps);
      for (int r=0;r<nx;r++) B[(size_t)r*nu+i]=ds[r]; } }
  memcpy(o->qpos,q0,8*nq); memcpy(o->qvel,v0,8*nv); memcpy(o->act,a0,8*na); memcpy(o->qacc_warmstart,w0,8*nv); memcpy(o->ctrl,ctrl,8*nu);
  o->time=t0; o->wrap_warm=ww0; memcpy(o->wrap_z,wz0,8*o->nwrap);
  free(q0); free(v0); free(a0); free(w0); free(wz0); free(f); free(x0); free(xp); free(xm); free(ds); free(q); free(v); free(a); free(e); free(c);
}
