"""Exact references for the 3 + m sums of one dual evaluation, the depth of every form's summation tree, the instance
families on which the parity tolerance of the older tests says nothing, and the wrong sums the check has to reject.
numpy and math.fsum only.

The per-variable terms come from tests/closed_form_model.py (pinned bit for bit to the oracle port and to the GPU), so
the exact sum of a returned value is math.fsum over known terms and the O(m) constants.  A kernel's value has to lie
within the rounding error of a float64 summation tree of known depth around it (check_dual_sums); the summation order
itself is not modelled.

tests/test_dual_sums.py pins the terms and the constants to the oracle port's sequential sums and shows that the check
rejects the wrong sums of mutants() on every instance; tests/test_dual_sums_gpu.py applies it to the library's kernels.
"""
import math

import numpy as np

import closed_form_model as cf
import outer_model as om
import synth

U = 2.0 ** -53
MMA, CCSAQ = cf.MMA, cf.CCSAQ
FOLD_THREADS = 256                      # chains of the folder CTA (fold_generation): records r, r + 256, ...


# ---- the depth of the summation trees -----------------------------------------------------------------------------------
def depth(form, g, m):
    """An upper bound on the number of rounded adds between one per-variable term and the kernel's sum, before the
    host adds the constant (nlopt_b200_dual_eval / nlopt_b200_dual_solve: one more add, counted by check_dual_sums).
    g: the one-rank geometry (outer_model.geometry); c = the most chunks in one group.

    "port" (the oracle port, mma.c:119-129): the terms are added in index order after the constant: n adds.

    "eval", "tma", "solve" (dual_eval_kernel via sweep_group, dual_eval_tma_kernel, and every solve kernel via
    sweep_group_preloaded or its TMA consumers): a thread holds one pair of every chunk of its group and adds the two
    terms of a pair one after the other (mma_pair / ccsaq_pair, or mma_point / ccsaq_point twice): 2 c adds from +0.0;
    warp_fold: 5 butterfly levels; put_group_record: the 8 warp records in warp order, 7 adds; fold_generation: chain t
    adds records t, t + 256, ... (ceil(P / 256) adds), warp_fold (5), then the 8 fold-warp results in warp order (7);
    the 8 virtual-shard sums in index order (eval_folder or solve_folder on one rank, publish_kernel on several): 7.
    Total 2 c + 31 + ceil(P / 256).

    "wide" (dual_eval_wide_kernel, m > 16): the val, g0 and w sums as above.  A constraint row: t = ta + tb (1),
    reduce8_rows (5 butterfly levels), one add per chunk into the warp's row sum wrow (c), the 8 warps' row sums in
    warp order (7), then the same fold: c + 32 + ceil(P / 256), never more than the first."""
    if form == "port":
        return int(g.n)
    c = int(np.diff(om.group_cuts(g)).max())
    fold = -(-int(g.groups_per_vshard) // FOLD_THREADS) + 5 + 7
    rows = 2 * c + 5 + 7
    if form == "wide":
        rows = max(rows, 1 + 5 + c + 7)
    elif form not in ("eval", "tma", "solve"):
        raise ValueError(form)
    return rows + fold + 7


# ---- the constants, in the order of nlopt_b200_dual_eval and the oracle port ------------------------------------------------
def constants(variant, inst, y):
    """(val, g0, w, gc[m]) starting values, None where nothing is added: val = f0 + y_0 c_0 + ... in index order, a
    NaN c_i counting as 0 under MMA (mma.c:75-78); g0 = f0; w: none; gc_i = c_i (0 for a NaN c_i under MMA).
    The sums returned are ret = -(val + S_val), g0 + S_g0, S_w, gc_i + S_gi."""
    y = np.asarray(y, dtype=np.float64)
    c0 = np.asarray(inst["c0"], dtype=np.float64)
    ci = np.where(np.isnan(c0), 0.0, c0) if variant == MMA else c0
    val = np.float64(inst["f0"])
    with np.errstate(all="ignore"):
        for i in range(inst["m"]):
            val = val + y[i] * ci[i]
    return [val, np.float64(inst["f0"]), None] + [np.float64(c) for c in ci]


def raw_values(out):
    """nlopt_b200_dual_eval's layout [ret, g0, w, gc...] -> the 3 + m values that are constant + sum (ret negated back)"""
    out = np.asarray(out, dtype=np.float64)
    return np.concatenate([[-out[0]], out[1:]])


class Sums:
    """What the 3 + m returned values may be, for term rows `terms` (one array per sum) and the constants `consts`
    (constants(), or None for a kernel's raw sums): the exact value of every sum, and the error a float64 summation
    tree of depth `dep` may add to it.  Computed once, then applied to any number of results (check, rejected)."""

    def __init__(self, terms, dep, consts=None):
        self.dep = dep
        self.k = len(terms)
        self.consts = [None] * self.k if consts is None else list(consts)
        self.want = []          # ("nan",) | ("inf", value) | ("num", exact, sum|t|, bound)
        for t, c in zip(terms, self.consts):
            t = np.asarray(t, dtype=np.float64)
            vals = t if c is None else np.append(t, c)
            if np.isnan(vals).any() or (np.isposinf(vals).any() and np.isneginf(vals).any()):
                self.want.append(("nan",))
            elif np.isinf(vals).any():
                self.want.append(("inf", float(vals[np.isinf(vals)][0])))
            else:
                a = math.fsum(np.abs(t).tolist())
                self.want.append(("num", math.fsum(vals.tolist()), a, self.bound(a, c)))

    def bound(self, abs_sum, const):
        """|got - exact| allowed for fl(const + S), S a summation tree of dep levels: gamma_dep sum|t| for the tree,
        u |const + S| for the last add, u |exact| for the rounding of fsum itself"""
        d = self.dep + 1 + (const is not None)
        c = 0.0 if const is None else 2.0 * abs(float(const))
        return (d * abs_sum + c) * U / (1.0 - d * U)

    def error(self, k, got):
        """None if `got` may be sum k; else why not"""
        w, got = self.want[k], float(got)
        if w[0] == "nan":
            return None if math.isnan(got) else f"a term is NaN, got {got!r}"
        if w[0] == "inf":
            return None if got == w[1] else f"a term is {w[1]!r}, got {got!r}"
        if not math.isfinite(got):
            return f"every term is finite, got {got!r}"
        if abs(got - w[1]) <= w[3]:
            return None
        return (f"got {got!r}, exact {w[1]!r}: {self.ratio(k, got):.3g} u sum|t| away, sum|t| {w[2]!r}, allowed {w[3]!r} "
                f"(depth {self.dep})")

    def ratio(self, k, got):
        """|got - exact| / (2^-53 sum|t|) of a finite sum k without a constant (or with +-0): what the summation tree
        costs.  0 where there is nothing to compare, and where the rounding of a nonzero constant's add is mixed in."""
        w = self.want[k]
        if w[0] != "num" or w[2] == 0.0 or (self.consts[k] is not None and self.consts[k] != 0.0):
            return 0.0
        return abs(float(got) - w[1]) / (U * w[2])

    def check(self, got, what=""):
        for k in range(self.k):
            err = self.error(k, got[k])
            assert err is None, f"{what}: sum {sum_name(k)}: {err}"

    def rejected(self, got):
        """the sums that check() would refuse"""
        return [k for k in range(self.k) if self.error(k, got[k]) is not None]

    def largest_ratio(self, got):
        return max(self.ratio(k, got[k]) for k in range(self.k))


def check_dual_sums(got, terms, dep, consts=None, what=""):
    """got: the 3 + m constant-plus-sum values (raw_values of what the library returned, or a probe's raw sums with
    consts None); terms: one array of terms per sum.  |got - fsum| <= (dep + 1) 2^-53 sum|t| (+ the constant's add);
    NaN exactly where a term or the constant is NaN."""
    Sums(terms, dep, consts).check(got, what)


def leading_constants(terms, consts):
    """the term rows with each constant in front: the sums of the oracle port, whose constant starts the chain and goes
    through every add after it"""
    return [t if c is None else np.append(np.float64(c), t) for t, c in zip(terms, consts)]


def sum_name(k):
    return ("val", "g0", "w")[k] if k < 3 else f"g_{k - 3}"


def term_rows(terms, has):
    return [terms[k][has[k]] for k in range(terms.shape[0])]


# ---- the exact sums and the wrong ones -------------------------------------------------------------------------------------
def apply_constants(raw, consts):
    """fl(const + S) for every sum, in the host's order"""
    out = np.empty(len(raw))
    with np.errstate(all="ignore"):
        for k, s in enumerate(raw):
            out[k] = s if consts[k] is None else consts[k] + np.float64(s)
    return out


def owners(g, n):
    """group and virtual shard of every variable"""
    cuts = om.group_cuts(g)
    grp = np.searchsorted(cuts, np.arange(n, dtype=np.int64) // om.CHUNK, side="right") - 1
    return grp, grp // int(g.groups_per_vshard)


def _fsum_by(values, keys, nkeys):
    order = np.argsort(keys, kind="stable")
    v, k = values[order], keys[order]
    edges = np.searchsorted(k, np.arange(nkeys + 1))
    return np.array([math.fsum(v[edges[s]:edges[s + 1]].tolist()) for s in range(nkeys)])


def mutants(variant, inst, g, y, y_prev):
    """Wrong results of one evaluation, in the constant-plus-sum layout: name -> 3 + m values, or None where the
    mutant cannot differ from the right result (terms that do not depend on y, fewer than two rows to swap).
    Each mutant takes the piece (variable, group, shard) whose terms are largest against sum|t|: a piece whose terms
    are below the rounding error of the whole sum is invisible to any tolerance, however tight."""
    n, m = inst["n"], inst["m"]
    _, terms, has = cf.evaluate(variant, inst, y)
    _, tprev, hprev = cf.evaluate(variant, inst, y_prev)
    consts = constants(variant, inst, y)
    with np.errstate(all="ignore"):
        T = np.where(has, terms, 0.0)
        Tp = np.where(hprev, tprev, 0.0)
    scale = np.array([math.fsum(np.abs(r).tolist()) if np.isfinite(r).all() else np.inf for r in T])
    scale = np.where(scale > 0, scale, 1.0)
    exact = np.array([math.fsum(r.tolist()) if np.isfinite(r).all() else np.nan for r in T])
    grp, vsh = owners(g, n)
    S = int(g.groups_total)

    def share(x):                                   # (3 + m, k) pieces -> the piece largest against sum|t| in some sum
        with np.errstate(all="ignore"):
            r = np.abs(x) / scale[:, None]
        return int(np.nanargmax(np.nanmax(np.where(np.isfinite(r), r, 0.0), axis=0)))

    out = {}
    finite = np.isfinite(T).all(axis=0)
    j = share(np.where(finite, T, 0.0))
    out["one variable's terms dropped"] = [math.fsum([exact[k], -T[k, j]]) for k in range(3 + m)]
    G = np.stack([_fsum_by(r, grp, S) if np.isfinite(r).all() else np.full(S, np.nan) for r in T])
    s = share(np.nan_to_num(G))
    out["one group record dropped"] = [math.fsum([exact[k], -G[k, s]]) for k in range(3 + m)]
    out["one group record counted twice"] = [math.fsum([exact[k], G[k, s]]) for k in range(3 + m)]
    V = np.stack([_fsum_by(r, vsh, 8) if np.isfinite(r).all() else np.full(8, np.nan) for r in T])
    v = share(np.nan_to_num(V))
    out["one virtual shard dropped"] = [math.fsum([exact[k], -V[k, v]]) for k in range(3 + m)]
    if not np.array_equal(T, Tp, equal_nan=True):   # no row, or every row switched off: the terms do not depend on y
        Gp = np.stack([_fsum_by(r, grp, S) if np.isfinite(r).all() else np.full(S, np.nan) for r in Tp])
        d = np.nan_to_num(np.abs(Gp - G))
        s2 = share(d)
        out["one group from the previous y"] = [math.fsum([exact[k], -G[k, s2], Gp[k, s2]]) for k in range(3 + m)]
    else:
        out["one group from the previous y"] = None
    if m >= 2:                                      # the kernel's sums of rows i and i + 1 in each other's slots
        i = int(np.argmax(np.nan_to_num(np.abs(exact[3:-1] - exact[4:]) / np.minimum(scale[3:-1], scale[4:]))))
        sw = list(exact)
        sw[3 + i], sw[4 + i] = exact[4 + i], exact[3 + i]
        out["g_i and g_i+1 swapped"] = sw
    else:
        out["g_i and g_i+1 swapped"] = None
    return {name: None if val is None else apply_constants(val, consts) for name, val in out.items()}


MUTANTS = ("one variable's terms dropped", "one group record dropped", "one group record counted twice",
           "one virtual shard dropped", "one group from the previous y", "g_i and g_i+1 swapped")


def previous_y(y):
    """the multipliers of the generation before: another point of the dual box"""
    y = np.asarray(y, dtype=np.float64)
    return 0.5 * y + 0.375


# ---- instance families -------------------------------------------------------------------------------------------------
FAMILIES = ("ordinary", "tiny sigma", "cancelling constants", "2^+-30 jumps", "uniform bounds", "fixed and unbounded",
            "NaN constraint value")


def instance(family, n, m, variant, seed=0):
    """an instance dict (tests/synth.py layout) of one family; f0 and c0 are set after the terms where they cancel"""
    s = synth.SEED0 + 7919 * seed + 101 * m + (n % 9973)
    inst = synth.kernel_instance(n, m, seed=s, special_lanes=family not in ("uniform bounds",))
    inst["c0"] = np.asarray(inst["c0"], dtype=np.float64).copy()
    if family == "tiny sigma":
        # sigma and the coordinates at 1e-9 (with x ~ 1, CCSAQ's dx ~ sigma^2 would vanish in x + dx); no constants:
        # fl(c + S) with c ~ 1 would hide the sums themselves
        for k in ("x", "lb", "ub", "sigma"):
            inst[k] = inst[k] * 1e-9
        inst["f0"] = 0.0
        inst["c0"][:] = 0.0
    elif family == "2^+-30 jumps":
        g = om.geometry(n)
        grp, vsh = owners(g, n)
        mid = int(g.groups_per_vshard) // 2               # a group boundary inside shard 0: groups mid - 1 | mid
        flip = (vsh + (grp >= mid) * (vsh == 0)) % 2
        k = np.where(flip == 0, 2.0 ** 30, 2.0 ** -30)
        inst["grad_f"] = inst["grad_f"] * k
        inst["grad_c"] = inst["grad_c"] * k[None, :]
    elif family == "fixed and unbounded":
        pick = (synth.u01(98, n, s) * 10).astype(np.int64)
        fixed = pick < 3
        inst["sigma"] = np.where(fixed, 0.0, inst["sigma"])
        inst["lb"] = np.where(fixed, inst["x"], np.where((pick == 3) | (pick == 5), -np.inf, inst["lb"]))
        inst["ub"] = np.where(fixed, inst["x"], np.where((pick == 4) | (pick == 5), np.inf, inst["ub"]))
    elif family == "NaN constraint value" and m:
        inst["c0"][1 if m > 1 else 0] = np.nan
    if family == "cancelling constants":
        _, terms, has = cf.evaluate(variant, inst)
        inst["f0"] = -math.fsum(terms[1][has[1]].tolist())
        for i in range(m):
            inst["c0"][i] = -math.fsum(terms[3 + i][has[3 + i]].tolist())
    return inst


def uniform_bounds(inst):
    return bool(np.all(inst["lb"] == inst["lb"][0]) and np.all(inst["ub"] == inst["ub"][0]))


def expected(variant, inst, y):
    """(x*, term rows, constants) of one evaluation at y"""
    xc, terms, has = cf.evaluate(variant, inst, y)
    return xc, term_rows(terms, has), constants(variant, inst, y)


# ---- the instances of the GPU test ---------------------------------------------------------------------------------------
MS = (0, 1, 2, 3, 4, 5, 8, 16)
# sizes: tiny and ragged; both sides of the first, a middle and the last two changes of groups_total below 3e6
# (tests/test_outer_kernels_gpu.geometry_edges); ragged shards of mid size
SIZES = (1, 3, 513, 4096, 4097, 100003, 110592, 110593, 221184, 221185, 1801729)
LARGE = ((MMA, 2, "2^+-30 jumps", 10 ** 7), (CCSAQ, 4, "uniform bounds", 10 ** 7))


def cases(variant, m, per=4):
    """(family, n) of the evaluation instances of one (variant, m): `per` of them, families and sizes dealt in turn so
    that every family meets every row count and most sizes over the whole set"""
    out = []
    base = 3 * MS.index(m) + 7 * variant
    for i in range(per):
        fam = FAMILIES[(base + i) % len(FAMILIES)]
        n = SIZES[(5 * base + 3 * i) % len(SIZES)]
        if fam == "NaN constraint value" and m == 0:
            fam = "ordinary"
        out.append((fam, n))
    out += [(fam, n) for v, mm, fam, n in LARGE if v == variant and mm == m]
    return out


def all_cases():
    return [(v, m, fam, n) for v in (MMA, CCSAQ) for m in MS for fam, n in cases(v, m)]


# the wide kernel: (m, n) with NaN constraint values on every seventh row in the second instance of each m
WIDE = ((17, 100003), (17, 4097), (37, 100003), (37, 513), (64, 20481), (257, 20481), (1000, 4097), (2048, 4097),
        (2048, 1025))


def wide_instance(m, n, variant, nan_rows):
    inst = instance("ordinary", n, m, variant, seed=1)
    if nan_rows:
        inst["c0"][3::7] = np.nan
    return inst
