"""``from_pymc(model)``: lower a ``pm.Model`` to ``pymc_b200.ir.ModelIR`` (SURVEY.md 8f-2, VERDICT r1 missing #1).

The reference hands a model to the sampler as one compiled callable over the raveled value variables
(``Model.logp_dlogp_function``, pymc/model/core.py:464-529).  This walks the same objects that callable is built from --
``model.free_RVs``, ``model.observed_RVs``, ``model.rvs_to_values``, ``model.rvs_to_transforms`` (core.py:406-409) and
each RV's owner node (the representation ``fgraph_from_model`` freezes into ``ModelFreeRV`` / ``ModelObservedRV`` nodes,
pymc/model/fgraph.py:76-81, :139) -- and pattern-matches them onto the closed factor set of the IR:

    free RV      ->  ir.Var (transform from rvs_to_transforms) + ir.Prior (parameters: constants or scalar free RVs;
                     a Normal / StudentT location may be any linear predictor -> ir.Linear, its sigma a constant vector),
                     AR(1) / GaussianRandomWalk -> ir.AR1
    observed RV  ->  ir.Likelihood; its location parameter is parsed into linear-predictor terms
                     (Add / Sub / Neg / Mul / division by a constant / indexing by constant integer arrays / Dot with a
                     constant matrix / broadcasts); Normal(0, exp(eta / 2)) with a linear eta -> the log-variance likelihood;
                     Binomial(n, logit_p = eta) with constant trials, NegativeBinomial(mu = exp(eta), alpha) and
                     Gamma(alpha, beta = alpha / exp(eta) | alpha * exp(-eta)), alpha a constant or a scalar free RV

Anything outside the closed set raises ``NotImplementedError`` naming the offending op, so a model either lowers exactly
or not at all.  PyMC and PyTensor are NOT importable in the build image (SURVEY 8c); this module imports them lazily and
tests/test_frontend.py runs under ``pytest.importorskip("pymc")``.
"""
from __future__ import annotations

import numpy as np

from . import ir as _ir

_PRIOR_BY_OP = {  # RV op class name (lower-cased, "rv" stripped) -> (ir dist, parameter indices in the op's dist params)
    "normal": ("normal", (0, 1)),
    "halfnormal": ("halfnormal", (1,)),   # (loc, sigma): loc must be 0
    "cauchy": ("cauchy", (0, 1)),
    "halfcauchy": ("halfcauchy", (1,)),   # (loc, beta)
    "exponential": ("exponential", (0,)),  # PyTensor's scale = 1 / lam: inverted below
    "studentt": ("studentt", (0, 1, 2)),
    "uniform": ("uniform", (0, 1)),
    "gamma": ("gamma", (0, 1)),           # (alpha, scale): beta = 1 / scale
    "beta": ("beta", (0, 1)),
    "lognormal": ("lognormal", (0, 1)),
    "flat": ("flat", ()),
    "halfflat": ("flat", ()),
}


def _op_name(rv) -> str:
    op = rv.owner.op
    name = type(op).__name__.lower()
    for suffix in ("rv",):
        if name.endswith(suffix):
            name = name[: -len(suffix)]
    return name


def _is_copy(node) -> bool:
    """A copy op of one input (what ``pm.Deterministic`` wraps its expression in, under some PyTensor versions)."""
    return type(node.op).__name__ in ("Identity", "Copy", "DeepCopyOp", "ViewOp") and len(node.inputs) == 1


def _dist_params(rv):
    op = rv.owner.op
    if hasattr(op, "dist_params"):
        return list(op.dist_params(rv.owner))
    return list(rv.owner.inputs[2:])  # legacy RandomVariable layout: rng, size, *params


def _const_value(x):
    """NumPy value of a graph node that does not depend on any random variable, else None."""
    from pytensor.graph.basic import Constant
    from pytensor.compile.sharedvalue import SharedVariable

    if isinstance(x, Constant):
        return np.asarray(x.data)
    if isinstance(x, SharedVariable):
        return np.asarray(x.get_value())
    try:
        from pymc.pytensorf import constant_fold

        return np.asarray(constant_fold([x], raise_not_constant=True)[0])
    except Exception:
        return None


def _static_size(x):
    """Number of elements of a graph variable when its type says so (``x.type.shape`` all known), else None."""
    shape = getattr(getattr(x, "type", None), "shape", None)
    if shape is None:
        shape = getattr(x, "static_shape", None)
    if shape is None or any(d is None for d in shape):
        return None
    return int(np.prod(shape, dtype=np.int64)) if len(shape) else 1


def from_pymc(model) -> _ir.ModelIR:
    import pymc as pm  # noqa: F401  (lazy: absent from the build image)
    from pytensor.tensor.elemwise import DimShuffle, Elemwise
    from pytensor.tensor.math import Dot
    from pytensor.tensor.subtensor import AdvancedSubtensor, AdvancedSubtensor1, Subtensor

    free = list(model.free_RVs)
    by_rv = {rv: model.rvs_to_values[rv] for rv in free}
    ip = model.initial_point()

    vars_, name_of = [], {}
    for rv in free:
        val = by_rv[rv]
        tr = model.rvs_to_transforms.get(rv)
        tname = type(tr).__name__.lower() if tr is not None else ""
        transform, bounds = None, None
        if tr is None:
            pass
        elif "log" in tname and "odds" not in tname and "interval" not in tname:
            transform = "log"
        elif "interval" in tname or "logodds" in tname:
            transform = "interval"
            if "logodds" in tname:
                bounds = (0.0, 1.0)
            else:
                lo, hi = tr.args_fn(*rv.owner.inputs)
                lo, hi = _const_value(lo), _const_value(hi)
                if lo is None or hi is None:
                    raise NotImplementedError(f"{rv.name}: interval transform with non-constant bounds")
                bounds = (float(lo), float(hi))
        else:
            raise NotImplementedError(f"{rv.name}: transform {type(tr).__name__} is outside the closed set (None, log, interval)")
        size = int(np.prod(ip[val.name].shape, dtype=np.int64)) if np.ndim(ip[val.name]) else 1
        vars_.append(_ir.Var(val.name, rv.name, size, transform, bounds, initial=np.ravel(ip[val.name]).astype(np.float64)))
        name_of[rv] = val.name
    size_of = {v.name: v.size for v in vars_}

    def param(x, what):
        if x in name_of:
            if size_of[name_of[x]] != 1:
                raise NotImplementedError(f"{what}: a vector random variable as a distribution parameter")
            return _ir.Ref(name_of[x])
        if x.owner is not None and isinstance(x.owner.op, DimShuffle) and x.owner.inputs[0] in name_of:
            return param(x.owner.inputs[0], what)
        v = _const_value(x)
        if v is None or v.size != 1:
            raise NotImplementedError(f"{what}: parameter is neither a constant scalar nor a scalar free RV")
        return float(v.reshape(()))

    # ---- linear predictors: likelihood locations, Linear prior locations, Deterministics ------------------------------
    def scalar_op_name(node):
        return type(node.op.scalar_op).__name__.lower() if isinstance(node.op, Elemwise) else ""

    def terms_of(x, N):
        """-> list of (coef: ndarray[N] | float, factors: [(var name, idx or None)])"""
        if x in name_of:
            return [(1.0, [(name_of[x], None)])]
        c = _const_value(x)
        if c is not None:
            c = np.broadcast_to(np.asarray(c, dtype=np.float64), (N,)).copy() if c.size > 1 else float(c.reshape(()))
            return [(c, [])]
        node = x.owner
        if node is None:
            raise NotImplementedError(f"linear predictor: free input {x} is not a model variable")
        if _is_copy(node) or scalar_op_name(node) == "identity":  # e.g. the named copy pm.Deterministic makes
            return terms_of(node.inputs[0], N)
        if isinstance(node.op, DimShuffle):
            return terms_of(node.inputs[0], N)
        if isinstance(node.op, (AdvancedSubtensor1, AdvancedSubtensor, Subtensor)):
            base, *ix = node.inputs
            if base in name_of and len(ix) == 1:
                iv = _const_value(ix[0])
                if iv is None:
                    raise NotImplementedError("linear predictor: indexing by a non-constant index")
                return [(1.0, [(name_of[base], np.broadcast_to(np.asarray(iv, dtype=np.int32), (N,)).copy())])]
            raise NotImplementedError("linear predictor: indexing of a non-variable expression")
        if isinstance(node.op, Dot):
            a, b = node.inputs
            A, B = _const_value(a), _const_value(b)
            if A is not None and b in name_of and A.ndim == 2:
                return [(np.ascontiguousarray(A[:, k], dtype=np.float64), [(name_of[b], np.full(N, k, dtype=np.int32))])
                        for k in range(A.shape[1])]
            raise NotImplementedError("linear predictor: dot() is supported as constant_matrix @ vector_variable")
        son = scalar_op_name(node)
        if son == "add":
            return [t for inp in node.inputs for t in terms_of(inp, N)]
        if son == "sub":
            a, b = node.inputs
            return terms_of(a, N) + [(-1.0 * c if np.ndim(c) == 0 else -c, f) for c, f in terms_of(b, N)]
        if son == "neg":
            return [(-1.0 * c if np.ndim(c) == 0 else -c, f) for c, f in terms_of(node.inputs[0], N)]
        if son in ("truediv", "true_div"):  # (linear predictor) / constant
            a, b = node.inputs
            d = _const_value(b)
            if d is None:
                raise NotImplementedError("linear predictor: division by a non-constant")
            d = np.broadcast_to(np.asarray(d, dtype=np.float64), (N,)).copy() if d.size > 1 else float(d.reshape(()))
            return [(c / d, f) for c, f in terms_of(a, N)]
        if son == "mul":
            acc = [(1.0, [])]
            for inp in node.inputs:
                nxt = []
                for c1, f1 in acc:
                    for c2, f2 in terms_of(inp, N):
                        if len(f1) + len(f2) > _ir.MAX_TERM_FACTORS:
                            raise NotImplementedError("linear predictor: a product of more than 3 random factors")
                        nxt.append((np.asarray(c1) * np.asarray(c2) if (np.ndim(c1) or np.ndim(c2)) else float(c1) * float(c2),
                                    f1 + f2))
                acc = nxt
            return acc
        raise NotImplementedError(f"linear predictor: op {node.op} is outside the closed set (add, sub, neg, mul, indexing, dot)")

    def make_terms(x, N):
        out = []
        for c, f in terms_of(x, N):
            coef = None if (np.ndim(c) == 0 and float(c) == 1.0) else (np.asarray(c, dtype=np.float64) if np.ndim(c) else float(c))
            out.append(_ir.Term(list(f), coef))
        return out

    priors, ar1 = [], []
    for rv in free:
        op = _op_name(rv)
        ps = _dist_params(rv)
        vn = name_of[rv]
        if op in ("autoregressive", "ar"):
            rhos, sigma = ps[0], ps[1]
            if int(getattr(rv.owner.op, "ar_order", 1)) != 1 or getattr(rv.owner.op, "constant_term", False):
                raise NotImplementedError(f"{rv.name}: only AR(1) without a constant term is in the closed set")
            init = ps[2]
            if _op_name(init) != "normal":
                raise NotImplementedError(f"{rv.name}: AR init_dist must be Normal(0, s)")
            ipar = _dist_params(init)
            if float(_const_value(ipar[0])) != 0.0:
                raise NotImplementedError(f"{rv.name}: AR init_dist must be centred at 0")
            rho = rhos.owner.inputs[0] if (rhos.owner is not None and not isinstance(rhos.owner.op, type(None)) and rhos not in name_of
                                           and _const_value(rhos) is None and len(rhos.owner.inputs) == 1) else rhos
            ar1.append(_ir.AR1(vn, param(rho, rv.name + ".rho"), param(sigma, rv.name + ".sigma"), float(_const_value(ipar[1]))))
            continue
        if op in ("gaussianrandomwalk", "randomwalk"):
            raise NotImplementedError(f"{rv.name}: write the random walk as pm.AR(rho=[1.0], ...) for this front-end")
        if op not in _PRIOR_BY_OP:
            raise NotImplementedError(f"{rv.name}: distribution {type(rv.owner.op).__name__} is outside the closed set "
                                      f"{sorted(_ir.PRIOR_DISTS)}")
        dist, idx = _PRIOR_BY_OP[op]
        loc, scale = _ir.LINEAR_PRIORS.get(dist, (None, None))

        def prior_arg(i):
            what = f"{rv.name}.param{i}"
            if i == loc:
                try:  # a constant or a scalar free RV; anything else is a linear predictor of the RV's size
                    return param(ps[i], what)
                except NotImplementedError:
                    return _ir.Linear(make_terms(ps[i], size_of[vn]))
            c = _const_value(ps[i]) if i == scale else None
            if c is not None and c.size > 1:  # one constant scale per element
                return np.ravel(np.broadcast_to(c, np.shape(ip[by_rv[rv].name]))).astype(np.float64)
            return param(ps[i], what)

        args = [prior_arg(i) for i in idx]
        if op in ("halfnormal", "halfcauchy"):
            c = _const_value(ps[0])
            if c is None or np.any(c != 0.0):
                raise NotImplementedError(f"{rv.name}: {op} with a non-zero location")
        if op == "exponential":  # PyTensor parametrises by scale = 1 / lam
            if isinstance(args[0], _ir.Ref):
                raise NotImplementedError(f"{rv.name}: Exponential with a random rate")
            args[0] = 1.0 / args[0]
        if op == "gamma":
            args[1] = 1.0 / args[1]
        priors.append(_ir.Prior(dist, vn, tuple(args)))

    # ---- observed RVs: likelihoods with a linear predictor ------------------------------------------------------------
    def strip(x, want):
        """peel one Elemwise layer named `want` (sigmoid / exp) off x, or return None"""
        if x.owner is not None and scalar_op_name(x.owner) == want:
            return x.owner.inputs[0]
        return None

    def inputs_of(x, want):
        """inputs of the Elemwise `want` (add / truediv / exp ...) that x is, under any DimShuffle layers, or None"""
        while x.owner is not None and isinstance(x.owner.op, DimShuffle):
            x = x.owner.inputs[0]
        if x.owner is not None and scalar_op_name(x.owner) == want:
            return list(x.owner.inputs)
        return None

    def same_param(x, p):
        """x (under DimShuffle layers) is the constant or scalar free RV p"""
        while x.owner is not None and isinstance(x.owner.op, DimShuffle):
            x = x.owner.inputs[0]
        try:
            return param(x, "") == p
        except NotImplementedError:
            return False

    liks = []
    for rv in model.observed_RVs:
        y = _const_value(model.rvs_to_values[rv])
        if y is None:
            raise NotImplementedError(f"{rv.name}: observed data must be constant")
        y = np.ravel(np.asarray(y, dtype=np.float64))
        N = len(y)
        op, ps = _op_name(rv), _dist_params(rv)

        def sigma_of(s):
            if s in name_of:
                return param(s, rv.name + ".sigma")
            v = _const_value(s)
            if v is not None:
                return float(v.reshape(())) if v.size == 1 else np.ravel(np.broadcast_to(v, (N,))).astype(np.float64)
            return param(s, rv.name + ".sigma")

        if op == "normal":
            # the stochastic-volatility observation y ~ Normal(0, exp(c * eta)) with a linear eta (c = 1/2: eta is the log-variance)
            log_sd, loc0 = ps[1], _const_value(ps[0])
            while log_sd.owner is not None and isinstance(log_sd.owner.op, DimShuffle):
                log_sd = log_sd.owner.inputs[0]
            log_sd = strip(log_sd, "exp")
            if log_sd is not None and loc0 is not None and not np.any(loc0):
                doubled = [(2.0 * c, f) for c, f in terms_of(log_sd, N)]  # eta = 2 log sd
                terms = [_ir.Term(list(f), None if (np.ndim(c) == 0 and float(c) == 1.0) else
                                  (np.asarray(c, dtype=np.float64) if np.ndim(c) else float(c))) for c, f in doubled]
                liks.append(_ir.Likelihood("normal_logvar", y, terms, name=rv.name))
                continue
            liks.append(_ir.Likelihood("normal", y, make_terms(ps[0], N), sigma=sigma_of(ps[1]), name=rv.name))
        elif op == "studentt":
            nu = _const_value(ps[0])
            if nu is None:
                raise NotImplementedError(f"{rv.name}: StudentT nu must be constant")
            liks.append(_ir.Likelihood("studentt", y, make_terms(ps[1], N), sigma=sigma_of(ps[2]), nu=float(nu), name=rv.name))
        elif op == "bernoulli":
            eta = strip(ps[0], "sigmoid")
            if eta is None:
                raise NotImplementedError(f"{rv.name}: write the likelihood as pm.Bernoulli(logit_p=...)")
            liks.append(_ir.Likelihood("bernoulli_logit", y, make_terms(eta, N), name=rv.name))
        elif op == "poisson":
            eta = strip(ps[0], "exp")
            if eta is None:
                raise NotImplementedError(f"{rv.name}: write the rate as pm.math.exp(linear predictor)")
            liks.append(_ir.Likelihood("poisson_log", y, make_terms(eta, N), name=rv.name))
        elif op == "binomial":  # RV parameters (n, p); logit_p= and p=invlogit(eta) both give p = sigmoid(eta)
            form = "pm.Binomial(n=trials, logit_p=linear predictor) with constant trials"
            nt = _const_value(ps[0])
            eta = inputs_of(ps[1], "sigmoid")
            if nt is None or eta is None:
                raise NotImplementedError(f"{rv.name}: write the likelihood as {form}")
            trials = float(nt.reshape(())) if nt.size == 1 else np.ravel(np.broadcast_to(nt, (N,))).astype(np.float64)
            liks.append(_ir.Likelihood("binomial_logit", y, make_terms(eta[0], N), trials=trials, name=rv.name))
        elif op in ("negbinomial", "nbinom"):  # RV parameters (n = alpha, p = alpha / (mu + alpha)), discrete.py:700-723
            form = "pm.NegativeBinomial(mu=pm.math.exp(linear predictor), alpha=constant or scalar free RV)"
            try:
                alpha = param(ps[0], rv.name + ".alpha")
            except NotImplementedError:
                raise NotImplementedError(f"{rv.name}: write the likelihood as {form}") from None
            div, eta = inputs_of(ps[1], "truediv"), None
            den = inputs_of(div[1], "add") if div is not None and same_param(div[0], alpha) else None
            if den is not None and len(den) == 2:
                for mu_, a_ in (den, den[::-1]):
                    e = inputs_of(mu_, "exp")
                    if e is not None and same_param(a_, alpha):
                        eta = e[0]
                        break
            if eta is None:
                raise NotImplementedError(f"{rv.name}: write the likelihood as {form}")
            liks.append(_ir.Likelihood("negative_binomial_log", y, make_terms(eta, N), alpha=alpha, name=rv.name))
        elif op == "gamma":  # RV parameters (alpha, scale = reciprocal(beta)), continuous.py:2478-2510
            form = ("pm.Gamma(alpha=a, beta=a / pm.math.exp(linear predictor)) or beta=a * pm.math.exp(-linear predictor), "
                    "a a constant or scalar free RV")
            try:
                alpha = param(ps[0], rv.name + ".alpha")
            except NotImplementedError:
                raise NotImplementedError(f"{rv.name}: write the likelihood as {form}") from None
            beta, eta = inputs_of(ps[1], "reciprocal"), None
            if beta is not None:
                div, mul = inputs_of(beta[0], "truediv"), inputs_of(beta[0], "mul")
                if div is not None and same_param(div[0], alpha):  # a / exp(eta)
                    e = inputs_of(div[1], "exp")
                    eta = e[0] if e is not None else None
                elif mul is not None and len(mul) == 2:  # a * exp(-eta), either order
                    for a_, e_ in (mul, mul[::-1]):
                        e = inputs_of(e_, "exp")
                        ng = inputs_of(e[0], "neg") if e is not None else None
                        if ng is not None and same_param(a_, alpha):
                            eta = ng[0]
                            break
            if eta is None:
                raise NotImplementedError(f"{rv.name}: write the likelihood as {form}")
            liks.append(_ir.Likelihood("gamma_log", y, make_terms(eta, N), alpha=alpha, name=rv.name))
        else:
            raise NotImplementedError(f"{rv.name}: likelihood {type(rv.owner.op).__name__} is outside the closed set "
                                      f"{sorted(_ir.LIK_DISTS)}")
    # ---- pm.Deterministic: recorded in the posterior, never part of logp -------------------------------------------------
    dets = []
    for dv in getattr(model, "deterministics", []) or []:
        size = _static_size(dv)
        if size is None:
            raise NotImplementedError(f"{dv.name}: the size of this Deterministic is not known statically")
        expr = dv
        if expr.owner is not None and _is_copy(expr.owner):
            expr = expr.owner.inputs[0]  # pm.Deterministic wraps its expression in a named copy
        terms = []
        for c, f in terms_of(expr, size):
            coef = None if (np.ndim(c) == 0 and float(c) == 1.0) else (np.asarray(c, dtype=np.float64) if np.ndim(c) else float(c))
            terms.append(_ir.Term(list(f), coef))
        dets.append(_ir.Deterministic(dv.name, size, terms))
    out = _ir.ModelIR(vars_, priors, liks, ar1, name=getattr(model, "name", "") or "pymc_model", deterministics=dets)
    out.validate()
    return out
