// nlopt_object.hpp -- the opaque object behind `nlopt_opt` in this library.
// Field meanings follow the reference's struct nlopt_opt_s (src/api/nlopt-internal.h:40-88);
// the layout is our own (the type is opaque across the ABI).
#pragma once

#include <string>
#include <vector>

#include "../../include/nlopt_b200.h"
#include "backend_factory.hpp"

namespace nb200 {

// one registered constraint object (reference: nlopt_constraint, src/util/nlopt-util.h:119-126)
struct ConstraintRec {
    FuncSpec fn;
    std::vector<double> tol;        // fn.m feasibility tolerances
};

struct NamedParam {
    std::string name;
    double val;
};

// device mode of one per-variable option (nlopt_b200_set_{xtol_abs,x_weights,initial_step}_device): its values live in
// dev (owned) and the option's host vector holds them only while mirror (after a host reader downloaded them); any host
// setter of that option frees dev
struct DeviceOption {
    DeviceVector *dev = nullptr;
    bool mirror = false;
};

}  // namespace nb200

struct nlopt_opt_s {
    nlopt_algorithm algorithm;
    unsigned n;

    nb200::FuncSpec objective;      // negate: while a maximisation with a device or sharded objective runs
    int maximize = 0;

    std::vector<nb200::NamedParam *> params;      // pointers stay valid: nlopt_nth_param hands out c_str()

    std::vector<double> lb, ub;
    bool lb_uniform = true, ub_uniform = true;   // every entry equal (set by nlopt_set_*_bounds1): filled on device
    // device mode (nlopt_b200_set_*_bounds_device): both bounds live in dbounds (owned) and lb / ub hold their values
    // only while lb_ub_mirror (after a host reader downloaded them); a host setter downloads them and leaves device mode
    nb200::DeviceBounds *dbounds = nullptr;
    bool lb_ub_mirror = false;
    std::vector<nb200::ConstraintRec> fc, h;      // inequality / equality constraint objects
    nlopt_munge munge_on_destroy = nullptr, munge_on_copy = nullptr;

    double stopval;
    double ftol_rel = 0, ftol_abs = 0, xtol_rel = 0;
    bool has_xtol_abs = false, has_x_weights = false, has_dx = false;
    std::vector<double> xtol_abs, x_weights, dx;
    nb200::DeviceOption xtol_abs_dev, x_weights_dev, dx_dev;     // has_* stays true in device mode
    int maxeval = 0, numevals = 0;
    double maxtime = 0;
    int force_stop = 0;
    nlopt_opt_s *force_stop_child = nullptr;

    nlopt_opt_s *local_opt = nullptr;
    const nb200::PenaltySpec *penalty = nullptr;  // set on the sub-optimiser while NLOPT_AUGLAG* drives it: its objective
                                                  // is the augmented Lagrangian built around f (never copied)
    unsigned stochastic_population = 0, vector_storage = 0;

    bool has_errmsg = false;
    std::string errmsg;

    nlopt_b200_stats stats{};
};
