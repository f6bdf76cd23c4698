// dual_machine_probe.cpp -- replays a recorded dual-optimiser trajectory into the host machine of
// nlopt_b200/csrc/dual_mma.hpp (DualMachine), the way DualMMA::solve drives it.  Tests only
// (tests/test_dual_machine.py builds it with the library's C++ flags, once per header mutant as well).
#include <cstring>

#include "dual_mma.hpp"

extern "C" {

// Start DualMachine on (m, y0, lo, hi, stop) and feed it the recorded F_k, grad F_k (ys, gs: K x m row-major) for as
// long as trial() equals ys[k] bit for bit.  From evaluation index k_time on (k_time < 0: never) the machine is told
// that the time limit has passed.  Returns the machine's result code; *status: 0 finished on the recorded answers,
// 1 trial point k != ys[k] (k in *where), 2 wanted more than K evaluations.
int dmp_replay(int m, const double *y0, const double *lo, const double *hi, const double *stop5, long k_time,
               long K, const double *ys, const double *fs, const double *gs,
               double *y_out, double *fmin_out, long *nevals_out, long *feeds_out, int *status, long *where)
{
    nb200::DualStop st{stop5[0], stop5[1], stop5[2], stop5[3], (int) stop5[4], k_time >= 0 ? 1.0 : 0.0};
    nb200::DualMachine mach;
    *status = 0;
    *where = -1;
    *feeds_out = 0;
    const int rc = mach.start(m, y0, lo, hi, st);
    if (rc != nb200::kRetSuccess) {
        *nevals_out = mach.nevals;
        return rc;
    }
    for (long k = 0;; ++k) {
        if (k == K) { *status = 2; *where = k; break; }
        if (std::memcmp(mach.trial(), ys + k * m, sizeof(double) * (size_t) m) != 0) { *status = 1; *where = k; break; }
        ++*feeds_out;
        if (mach.feed(fs[k], gs + k * m, k_time >= 0 && k >= k_time ? 1.0 : 0.0)) break;
    }
    for (int i = 0; i < m; ++i) y_out[i] = mach.y[i];
    *fmin_out = mach.fmin;
    *nevals_out = mach.nevals;
    return mach.ret;
}

}
