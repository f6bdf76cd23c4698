/* jit_simp.c -- SIMP compliance + volume under LD_MMA from plain C: the functors are source strings compiled by the
 * library at run time (nlopt_b200_jit_create), so this program needs gcc, include/nlopt_b200.h and -lnlopt_b200 only.
 * Prints the result code, the number of evaluations and the bits of f* (hex, most significant byte first). */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "nlopt_b200.h"

static const char *kSource =
    "__device__ inline unsigned long long mix64(unsigned long long z)\n"
    "{\n"
    "    z += 0x9E3779B97F4A7C15ull;\n"
    "    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;\n"
    "    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;\n"
    "    return z ^ (z >> 31);\n"
    "}\n"
    "__device__ inline double u01(unsigned long long seed, unsigned k, unsigned long long j)\n"
    "{\n"
    "    return (double) (mix64((seed + k) * 0x9E3779B97F4A7C15ull + j) >> 11) * 0x1.0p-53;\n"
    "}\n"
    "struct Simp {                   /* f(x) = sum_j a_j / (eps + (1 - eps) x_j^3) */\n"
    "    unsigned long long seed;\n"
    "    double eps;\n"
    "    __device__ double operator()(unsigned long long j, unsigned long long, long long jl, long long,\n"
    "                                 const double *x, double *grad_j) const\n"
    "    {\n"
    "        const double a = __dadd_rn(0.5, u01(seed, 0, j));\n"
    "        const double xj = x[jl], x2 = __dmul_rn(xj, xj), x3 = __dmul_rn(x2, xj);\n"
    "        const double ome = __dsub_rn(1.0, eps);\n"
    "        const double d = __dadd_rn(eps, __dmul_rn(ome, x3));\n"
    "        if (grad_j) *grad_j = -__ddiv_rn(__dmul_rn(__dmul_rn(a, __dmul_rn(ome, 3.0)), x2), __dmul_rn(d, d));\n"
    "        return __ddiv_rn(a, d);\n"
    "    }\n"
    "};\n"
    "struct Volume {                 /* mean(x) - 0.4: terms x_j, finish on the host */\n"
    "    double inv_n, offset;\n"
    "    __device__ double operator()(unsigned long long, unsigned long long, long long jl, long long,\n"
    "                                 const double *x, double *grad_j) const\n"
    "    {\n"
    "        if (grad_j) *grad_j = inv_n;\n"
    "        return x[jl];\n"
    "    }\n"
    "};\n";

/* the host sides of the functors: the same members in the same order */
struct Simp { unsigned long long seed; double eps; };
struct Volume { double inv_n, offset; };

static double volume_finish(double total, void *data)
{
    const struct Volume *v = (const struct Volume *) data;
    return total * v->inv_n + v->offset;
}

static nlopt_b200_jit compile(const char *name)
{
    nlopt_b200_jit h = nlopt_b200_jit_create(kSource, name, NULL, 0);
    if (!h || nlopt_b200_jit_errmsg(h)) {
        fprintf(stderr, "%s: %s\n", name, h ? nlopt_b200_jit_errmsg(h) : "out of memory");
        exit(1);
    }
    return h;
}

int main(void)
{
    const unsigned n = 20011;
    nlopt_b200_jit simp = compile("Simp"), volume = compile("Volume");
    struct Simp sp = {0x5EED0000ull, 1e-3};
    struct Volume vp = {1.0 / (double) n, -0.4};

    nlopt_opt opt = nlopt_create(NLOPT_LD_MMA, n);
    nlopt_set_lower_bounds1(opt, 1e-3);
    nlopt_set_upper_bounds1(opt, 1.0);
    nlopt_set_maxeval(opt, 12);
    if (nlopt_b200_jit_set_min_objective(opt, simp, &sp, sizeof sp, NULL, NULL) < 0
        || nlopt_b200_jit_add_inequality_constraint(opt, volume, &vp, sizeof vp, volume_finish, &vp, 1e-8) < 0) {
        fprintf(stderr, "registration: %s\n", nlopt_get_errmsg(opt));
        return 1;
    }
    double *x = malloc(n * sizeof(double)), f = 0.0;
    for (unsigned j = 0; j < n; ++j) x[j] = 0.5;
    const nlopt_result ret = nlopt_optimize(opt, x, &f);
    unsigned long long bits;
    memcpy(&bits, &f, sizeof bits);
    printf("%d %d %016llx\n", (int) ret, nlopt_get_numevals(opt), bits);
    nlopt_destroy(opt);             /* the opt first: the handles own its registrations */
    nlopt_b200_jit_destroy(simp);
    nlopt_b200_jit_destroy(volume);
    free(x);
    return ret > 0 ? 0 : 1;
}
