// C entry points on the host palette builder of the sigma index (nlopt_b200/csrc/sigma_palette.hpp), for
// tests/test_sigma_palette.py.  Built with g++ into tests/_build/ by that test; no GPU involved.
#include "../../nlopt_b200/csrc/sigma_palette.hpp"

extern "C" {

// Palette after `updates` sigma updates.  sizes[k] = entries (padding entry included) after k + 1 updates; val / next
// receive the final palette when non-null (capacity `cap` entries).  Returns the number of updates that fit the cap.
int nb200_sigma_palette(double lb, double ub, double init, double kappa, double sigma_min, int updates, long long *sizes,
                        double *val, unsigned short *next, long long cap, long long *nval, long long *nrows)
{
    nb200::SigmaPalette p;
    p.reset(nb200::SigmaPalette::sigma0(lb, ub, init, sigma_min), lb, ub, kappa, sigma_min);
    int done = 0;
    for (; done < updates; ++done) {
        if (!p.step()) break;
        if (sizes) sizes[done] = (long long) p.val.size();
    }
    *nval = (long long) p.val.size();
    *nrows = (long long) p.rows();
    if (val && (long long) p.val.size() <= cap) {
        for (size_t i = 0; i < p.val.size(); ++i) val[i] = p.val[i];
        for (size_t i = 0; i < p.next.size(); ++i) next[i] = p.next[i];
    }
    return done;
}

long long nb200_sigma_palette_cap() { return (long long) nb200::SigmaPalette::kCap; }
}
