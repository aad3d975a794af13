// tests/fp_exact/fp_exact.cpp — TEST INFRASTRUCTURE ONLY.
// The FP64 path's modular primitives and its generic transform, compiled for the host from the product headers unchanged
// (with -ffp-contract=off, so DMUL / DFMA / DADD stay separate IEEE operations as on the device), behind batch entry points
// that tests/test_fp_exact.py checks against exact integers.  Nothing here is part of the product library.
#include <cmath>
#include <cstring>
#include <vector>

// pass-output audit of the transform (ntt_fp_body.cuh B200_FP_AUDIT): largest |x| per pass in execution order, and a count
// of values that are not integers
static int g_logn, g_np, g_L[8];
static double g_amax[8];
static long long g_nonint;
static int fpx_audit_step(bool fwd, int logs)
{
    int acc = 0;
    for (int s = 0; s < g_np; s++)
    {
        const int pi = fwd ? s : g_np - 1 - s;
        if ((fwd ? g_logn - acc - g_L[pi] : acc) == logs)
            return s;
        acc += g_L[pi];
    }
    return 7;
}
static inline void fpx_audit(bool fwd, int logs, double x)
{
    const int s = fpx_audit_step(fwd, logs);
    if (std::fabs(x) > g_amax[s])
        g_amax[s] = std::fabs(x);
    if (x != std::nearbyint(x))
        g_nonint++;
}
#define B200_FP_AUDIT(fwd, logs, x) fpx_audit((fwd), (logs), (x))

#include "../../sunscreen_b200/csrc/modarith.cuh"
#include "../../sunscreen_b200/csrc/ntt_fp_body.cuh"

typedef long long i64;

extern "C" {

// kind 0: fp_mulmod, 1: fp_mulmod_x, 2: fp_mulmod_term(0, ..), 3: fp_mulmod_term(1, ..)
void fpx_mulmod(int kind, i64 cnt, const double *y, const double *w, const double *wp, double p, double *out)
{
    for (i64 i = 0; i < cnt; i++)
        out[i] = kind == 0 ? fp_mulmod(y[i], w[i], wp[i], p)
                 : kind == 1 ? fp_mulmod_x(y[i], w[i], wp[i], p)
                             : fp_mulmod_term(kind - 2, y[i], w[i], wp[i], p);
}

void fpx_mulmod2(i64 cnt, const double *a, const double *b, double p, double pinv, double *out)
{
    for (i64 i = 0; i < cnt; i++)
        out[i] = fp_mulmod2(a[i], b[i], p, pinv);
}

// xu 0: fp_renorm, 1: fp_renorm_x
void fpx_renorm(int xu, i64 cnt, const double *x, double p, double pinv, double *out)
{
    for (i64 i = 0; i < cnt; i++)
        out[i] = xu ? fp_renorm_x(x[i], p, pinv) : fp_renorm(x[i], p, pinv);
}

void fpx_to_canonical(int xu, i64 cnt, const double *x, double p, double pinv, u64 *out)
{
    for (i64 i = 0; i < cnt; i++)
        out[i] = xu ? fp_to_canonical<true>(x[i], p, pinv) : fp_to_canonical<false>(x[i], p, pinv);
}

// the bookkeeping's bounds: fp_prod_bound(p, |y[i]|) per operand, fp_renormed_bound(p)
void fpx_prod_bound(i64 cnt, double p, const double *y, double *out)
{
    for (i64 i = 0; i < cnt; i++)
        out[i] = fp_prod_bound(p, std::fabs(y[i]));
}
double fpx_renormed_bound(double p) { return fp_renormed_bound(p); }

// an inner product of K terms as the BEHZ kernels form it (bfv_body.cuh lift_coeff_fp / scale_coeff_fp): the first term
// with fp_mulmod, term i >= 1 with fp_mulmod_term(i - 1, ..), summed with DADD; partial[c*K + i] is the sum after term i,
// renormed[c] = fp_renorm of the sum, canon[c] = fp_to_canonical of the sum
void fpx_inner(i64 cnt, int K, const double *y, const double *w, const double *wp, double p, double pinv, double *partial,
               double *renormed, u64 *canon)
{
    for (i64 c = 0; c < cnt; c++)
    {
        const double *yc = y + c * K, *wc = w + c * K, *wpc = wp + c * K;
        double acc = fp_mulmod(yc[0], wc[0], wpc[0], p);
        partial[c * K] = acc;
        for (int i = 1; i < K; i++)
        {
            acc = B200_DADD(acc, fp_mulmod_term(i - 1, yc[i], wc[i], wpc[i], p));
            partial[c * K + i] = acc;
        }
        renormed[c] = fp_renorm(acc, p, pinv);
        canon[c] = fp_to_canonical(acc, p, pinv);
    }
}

// the generic FP64 transform (ntt_fp_block_body: the group routine the statically scheduled kernels run too) of `count`
// polynomials in place, with the forward pass schedule L[0..np) and the given renorm masks.  tw_fwd / tw_inv: the n twiddles
// (bit-reversed powers of the root and their inverses), inv_n / inv_n_w: n^-1 and n^-1 * tw_inv[1].  amax[0..np): the
// largest |x| each pass wrote, in execution order; returns the number of non-integer values written.
i64 fpx_ntt(int forward, int logn, int np, const int *L, double p, const double *tw_fwd, const double *tw_inv, double inv_n,
            double inv_n_w, unsigned renorm_fwd, unsigned renorm_inv, u64 *data, i64 count, double *amax)
{
    const int n = 1 << logn;
    NttPrimeFp P;
    std::memset(&P, 0, sizeof(P));
    P.p = p;
    P.pinv = 1.0 / p;
    P.inv_n[0] = inv_n;
    P.inv_n[1] = inv_n / p;
    P.inv_n_w[0] = inv_n_w;
    P.inv_n_w[1] = inv_n_w / p;
    P.fwd = tw_fwd;
    P.inv = tw_inv;
    P.renorm_fwd = renorm_fwd;
    P.renorm_inv = renorm_inv;
    P.enabled = 1;
    NttPrime PI;
    std::memset(&PI, 0, sizeof(PI));
    PI.p = (u64)p;
    NttJob job;
    std::memset(&job, 0, sizeof(job));
    job.logn = logn;
    job.npass = np;
    for (int i = 0; i < np; i++)
        job.pass_L[i] = L[i];
    g_logn = logn;
    g_np = np;
    for (int i = 0; i < 8; i++)
    {
        g_L[i] = i < np ? L[i] : 0;
        g_amax[i] = 0;
    }
    g_nonint = 0;
    std::vector<double> smd(ntt_smem_words(n));
    for (i64 c = 0; c < count; c++)
    {
        u64 *poly = data + c * n;
        if (forward)
            ntt_fp_block_body<true>(job, P, PI, poly, poly, smd.data(), 0, 1);
        else
            ntt_fp_block_body<false>(job, P, PI, poly, poly, smd.data(), 0, 1);
    }
    for (int i = 0; i < np; i++)
        amax[i] = g_amax[i];
    return g_nonint;
}

void fpx_shoup(int lazy, i64 cnt, const u64 *y, const u64 *w, const u64 *wq, u64 q, u64 *out)
{
    for (i64 i = 0; i < cnt; i++)
        out[i] = lazy ? shoup_mul_lazy(y[i], w[i], wq[i], q) : shoup_mul(y[i], w[i], wq[i], q);
}

void fpx_barrett64(i64 cnt, const u64 *x, u64 q, u64 ratio1, u64 *out)
{
    for (i64 i = 0; i < cnt; i++)
        out[i] = barrett64(x[i], q, ratio1);
}

void fpx_barrett128(i64 cnt, const u64 *lo, const u64 *hi, u64 q, u64 r0, u64 r1, u64 *out)
{
    for (i64 i = 0; i < cnt; i++)
        out[i] = barrett128(lo[i], hi[i], q, r0, r1);
}

// op 0: add_mod, 1: sub_mod, 2: neg_mod (b unused)
void fpx_addsub(int op, i64 cnt, const u64 *a, const u64 *b, u64 q, u64 *out)
{
    for (i64 i = 0; i < cnt; i++)
        out[i] = op == 0 ? add_mod(a[i], b[i], q) : op == 1 ? sub_mod(a[i], b[i], q) : neg_mod(a[i], q);
}
}
