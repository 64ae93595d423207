/* TEST INFRASTRUCTURE (oracle/): host check of the cached-reciprocal division of the specialised RK4 kernel
 * (parcels_b200/csrc/common.cuh div_by_cached): q = a r, two residual corrections with r = RN(1 / b), against the division
 * itself, on bcoord-like operands, random mantissas, the two constant divisors of the hot path (deg2m = 111120, 6) and quotients
 * built next to rounding midpoints.  tests/test_oracle_c.py builds and runs it (gcc -O2 -mfma -ffp-contract=off).
 * The primary check is tests/test_gpu_math.py, which runs the device function itself (pb_debug_math) on the same distributions;
 * this host copy is the larger stress run. */
/*
 * Prints "n=... bad3=... bad5=..." (bad3: a single correction step, for reference); exit status 1 when bad5 != 0. */
#include <math.h>
#include <stdio.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
static uint64_t s[2]={0x9E3779B97F4A7C15ULL,0xD1B54A32D192ED03ULL};
static inline uint64_t nxt(){uint64_t a=s[0],b=s[1];s[0]=b;a^=a<<23;s[1]=a^b^(a>>17)^(b>>26);return s[1]+b;}
static inline double u01(){return (nxt()>>11)*(1.0/9007199254740992.0);}
static inline double div5(double a,double b,double r){double q=a*r;double e=fma(-b,q,a);q=fma(e,r,q);e=fma(-b,q,a);q=fma(e,r,q);return q;}
static inline double div3(double a,double b,double r){double q=a*r;double e=fma(-b,q,a);q=fma(e,r,q);return q;}
int main(int argc,char**argv){
  long n=argc>1?atol(argv[1]):100000000L; long bad3=0,bad5=0;
  for(long i=0;i<n;i++){
    double a,b; int mode=i&7;
    if(mode<3){ b=ldexp(1.0+u01(), (int)(nxt()%40)-20); a=b*u01(); }          /* bcoord-like: 0<a<=b */
    else if(mode<5){ uint64_t x=nxt(),y=nxt(); x=(x&0x000FFFFFFFFFFFFFULL)|((uint64_t)(1023-30+(nxt()%60))<<52); y=(y&0x000FFFFFFFFFFFFFULL)|((uint64_t)(1023-30+(nxt()%60))<<52); memcpy(&a,&x,8); memcpy(&b,&y,8);} /* random mantissas */
    else if(mode==5){ b=111120.0; a=ldexp(1.0+u01(),(int)(nxt()%60)-50)*(nxt()&1?-1:1); }
    else if(mode==6){ b=6.0; a=ldexp(1.0+u01(),(int)(nxt()%60)-50)*(nxt()&1?-1:1); }
    else { /* adversarial: quotient near a midpoint: pick q midpoint-ish, b random, a=RN(q*b) */
      double q=1.0+u01(); uint64_t qi; memcpy(&qi,&q,8); double qn; uint64_t qj=qi+1; memcpy(&qn,&qj,8); double mid=0.5*(q+qn); /* inexact mid rounds, fine */
      b=1.0+u01(); a=mid*b; (void)qn; }
    double r=1.0/b; double t=a/b;
    if(div3(a,b,r)!=t) bad3++;
    if(div5(a,b,r)!=t) bad5++;
  }
  printf("n=%ld bad3=%ld bad5=%ld\n",n,bad3,bad5); return bad5!=0;}
