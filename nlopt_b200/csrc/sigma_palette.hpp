// sigma_palette.hpp -- every value sigma_j can take in one run, when it is a function of the update count and branches only.
//
// With uniform bounds and a uniform initial step, sigma_init_kernel gives every variable the same sigma_0, and each
// sigma update of end_outer_kernel (mma.c:431-442, ccsa_quadratic.c:577-590) applies one of three maps to sigma_j:
//   F_b(s) = max(clamp(s * gamma_b, kappa * range, 10 * range), sigma_min),   gamma = {0.7, 1.2, 1.0}
// (no clamp when a bound is infinite).  So after k updates sigma_j lies in the closure P_k of sigma_0 under the three
// maps, which does not depend on the data and grows polynomially in k (|P_7| = 68 at kappa = 1e-8 on [-2, 2]).  The
// palette is the union of P_0 .. P_k with stable indices: entry 0 is 0.0 (the padding lanes), entry 1 sigma_0, and
// next[3 i + b] is the index of F_b(val[i]).  The dual kernels then read a 16-bit index per variable instead of 8 bytes.
//
// F_b is evaluated with the operations of end_outer_kernel in the same order: single IEEE multiplies, subtractions and
// compares, which no compiler contracts (the library is built with -ffp-contract=off), so val[] has the device's bits.
#pragma once

#include <cmath>
#include <cstdint>
#include <cstring>
#include <unordered_map>
#include <vector>

#ifndef NB200_SIGMA_PALETTE_CAP
#define NB200_SIGMA_PALETTE_CAP 65535      // entries, padding entry included: every index fits 16 bits
#endif

namespace nb200 {

struct SigmaPalette {
    static constexpr size_t kCap = NB200_SIGMA_PALETTE_CAP;
    static_assert(kCap >= 2 && kCap <= 65536, "palette indices are 16-bit");

    std::vector<double> val;          // val[0] = 0.0 (padding lanes), val[1] = sigma_0
    std::vector<uint16_t> next;       // next[3 i + b], b = 0: x0.7, 1: x1.2, 2: x1 -- rows of the first rows() entries
    size_t rows() const { return next.size() / 3; }

    // sigma_0 as sigma_init_kernel computes it for uniform bounds and a uniform initial step (init, or none: <= 0)
    static double sigma0(double lb, double ub, double init, double sigma_min)
    {
        double s;
        if (init > 0) s = init;
        else if (std::isinf(ub) || std::isinf(lb)) s = 1.0;
        else s = 0.5 * (ub - lb);
        return s > sigma_min ? s : sigma_min;
    }

    void reset(double sigma_0, double lb, double ub, double kappa, double sigma_min)
    {
        lb_ = lb; ub_ = ub; kappa_ = kappa; sigma_min_ = sigma_min;
        val.assign(1, 0.0);
        next.assign(3, 0);
        where_.clear();
        add(sigma_0);
    }

    // the maps of end_outer_kernel, branch b as there: osc < 0 -> 0, osc > 0 -> 1, otherwise (0 or NaN) -> 2
    double map(double s, int b) const
    {
        s = s * (b == 0 ? 0.7 : b == 1 ? 1.2 : 1.0);
        if (!std::isinf(ub_) && !std::isinf(lb_)) {
            const double range = ub_ - lb_;
            const double top = 10.0 * range, bot = kappa_ * range;
            s = s < top ? s : top;
            s = s > bot ? s : bot;
        }
        return s > sigma_min_ ? s : sigma_min_;
    }

    // one more sigma update: the rows of the entries that have none yet, and the new values they reach.  False (and the
    // palette unusable) when that would take it past kCap entries.
    bool step()
    {
        const size_t end = val.size();
        for (size_t i = rows(); i < end; ++i)
            for (int b = 0; b < 3; ++b) {
                const double v = map(val[i], b);
                uint64_t key;
                std::memcpy(&key, &v, sizeof key);
                auto it = where_.find(key);
                if (it == where_.end()) {
                    if (val.size() >= kCap) return false;
                    it = where_.emplace(key, (uint16_t) val.size()).first;
                    val.push_back(v);
                }
                next.push_back(it->second);
            }
        return true;
    }

private:
    void add(double v)
    {
        uint64_t key;
        std::memcpy(&key, &v, sizeof key);
        where_.emplace(key, (uint16_t) val.size());
        val.push_back(v);
    }
    double lb_ = 0, ub_ = 0, kappa_ = 0, sigma_min_ = 0;
    std::unordered_map<uint64_t, uint16_t> where_;      // value bits -> index; the padding entry is not in it
};

}  // namespace nb200
