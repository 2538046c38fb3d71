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
                     Gamma(alpha, beta = alpha / exp(eta) | alpha * exp(-eta)), alpha a constant or a scalar free RV;
                     pm.Censored(pm.Normal.dist(eta, sigma), lower, upper), pm.TruncatedNormal(eta, sigma, lower, upper)
                     and pm.Truncated(pm.Normal.dist(eta, sigma), lower, upper) with constant bounds;
                     survival: pm.Weibull(alpha, beta=exp(eta)), pm.Exponential(scale=exp(eta)) or (lam=exp(-eta)) (the
                     Weibull with alpha = 1) and pm.LogNormal(eta, sigma), plain, or under pm.Censored / pm.Truncated with
                     constant bounds;
                     Beta regression: pm.Beta(mu=invlogit(eta), nu=phi) or pm.Beta(alpha=mu * phi, beta=(1 - mu) * phi)
                     and pm.BetaBinomial(alpha=mu * phi, beta=(1 - mu) * phi, n=trials) with constant trials, mu =
                     invlogit(eta), phi a constant or a scalar free RV;
                     pm.OrderedLogistic / pm.OrderedProbit: the Categorical whose p is their compute_p graph, with or
                     without the {name}_probs Deterministic (recorded, evaluated from the draws);
                     pm.ZeroInflatedPoisson / Binomial / NegativeBinomial and pm.HurdlePoisson / NegativeBinomial / Gamma:
                     the mixture of DiracDelta(0) and the family above with weights stack([1 - psi, psi]), psi a
                     constant, a scalar free RV or pm.math.invlogit(linear predictor);
                     finite mixtures: pm.NormalMixture(w, mu, sigma) and pm.Mixture(w, pm.Poisson.dist(lam, shape=K)), the
                     Mixture of ONE batched component, with w a free pm.Dirichlet or a constant K-vector, mu optionally
                     linear_predictor[:, None] + mu and lam optionally pm.math.exp(linear_predictor)[:, None] * lam
                 Gaussian processes: phi @ (beta * sqrt_psd), what pm.gp.HSGP.prior (non-centred) and prior_linearized
                     build, with psd cov.py's ExpQuad / Matern52 / Matern32 density, optionally times eta**2 (eta a scalar
                     free RV) or a constant, ls constants or a scalar or vector free RV -> an ir.Spectral term
    free RV      ->  pm.Dirichlet with a constant a -> the dirichlet prior on a simplex variable; pm.InverseGamma with
                     constant alpha, beta
    transform    ->  None, log, interval, Ordered() / Ordered(positive=True) -> "ordered" / "ordered_positive", and
                     SimplexTransform -> "simplex"

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
    "invgamma": ("inversegamma", (0, 1)),  # pm.InverseGamma's InvGammaRV: (alpha, beta) = (shape, scale), continuous.py:2593-2640
    "flat": ("flat", ()),
    "halfflat": ("flat", ()),
}


class _SpectralCoef:
    """The coefficient slot of an HSGP term in ``terms_of``: Phi with its ``ir.Spectral``.  Such a term may only be added
    to a predictor; scaling or negating it raises."""

    def __init__(self, Phi, spectral):
        self.Phi, self.spectral = Phi, spectral

    def _refuse(self, *args):
        raise NotImplementedError("linear predictor: an HSGP term phi @ (beta * sqrt_psd) may only be added, not scaled, "
                                  "negated or multiplied")

    __array__ = __float__ = __neg__ = __mul__ = __rmul__ = __truediv__ = _refuse


HSGP_FORM = ("pm.gp.HSGP(m, c, cov_func=eta**2 * pm.gp.cov.ExpQuad | Matern52 | Matern32(D, ls)).prior (non-centred), "
             "or phi @ (beta * sqrt_psd) from prior_linearized")


def _op_name(rv) -> str:
    return _op_class_name(rv.owner.op)


def _op_class_name(op) -> str:
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
        elif tname == "chain":
            raise NotImplementedError(f"{rv.name}: Chain([...]) transforms are outside the closed set (None, log, interval, "
                                      "ordered)")
        elif tname == "ordered":  # Ordered(positive, ascending), transforms.py:79-120
            if not getattr(tr, "ascending", True):
                raise NotImplementedError(f"{rv.name}: Ordered(ascending=False) is outside the closed set (only ascending "
                                          "ordered transforms)")
            transform = "ordered_positive" if getattr(tr, "positive", False) else "ordered"
        elif tname == "simplextransform":  # transforms.py:1091-1116: the value variable has K - 1 elements
            transform = "simplex"
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
    simplex = {v.name for v in vars_ if v.transform == "simplex"}

    def use(x):
        """the value variable of free RV x, which may enter any factor except a simplex (Dirichlet) one"""
        if name_of[x] in simplex:
            raise NotImplementedError(f"{x.name}: {_ir.SIMPLEX_USE} (pm.NormalMixture / pm.Mixture w)")
        return name_of[x]

    def param(x, what):
        if x in name_of:
            use(x)
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
            return [(1.0, [(use(x), None)])]
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
                return [(1.0, [(use(base), np.broadcast_to(np.asarray(iv, dtype=np.int32), (N,)).copy())])]
            raise NotImplementedError("linear predictor: indexing of a non-variable expression")
        if isinstance(node.op, Dot):
            a, b = node.inputs
            A, B = _const_value(a), _const_value(b)
            if A is not None and b in name_of and A.ndim == 2:
                return [(np.ascontiguousarray(A[:, k], dtype=np.float64), [(use(b), np.full(N, k, dtype=np.int32))])
                        for k in range(A.shape[1])]
            found = hsgp_of(b, A) if A is not None and A.ndim == 2 else None
            if found is not None and isinstance(found[1], np.ndarray):  # constant sqrt_psd: the design term Phi diag(s)
                return [(np.ascontiguousarray(A * found[1][None, :], dtype=np.float64), [(use(found[0]), None)])]
            if found is not None:
                return [(_SpectralCoef(np.ascontiguousarray(A, dtype=np.float64), found[1]), [(use(found[0]), None)])]
            raise NotImplementedError("linear predictor: dot() is supported as constant_matrix @ vector_variable or "
                                      f"an HSGP term ({HSGP_FORM})")
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
            if isinstance(c, _SpectralCoef):
                out.append(_ir.Term(list(f), c.Phi, spectral=c.spectral))
                continue
            coef = None if (np.ndim(c) == 0 and float(c) == 1.0) else (np.asarray(c, dtype=np.float64) if np.ndim(c) else float(c))
            out.append(_ir.Term(list(f), coef))
        return out

    # ---- HSGP: phi @ (beta * sqrt(psd)) with psd as cov.py's power_spectral_density builds it --------------------------
    def unshuffle(x):
        while x.owner is not None and isinstance(x.owner.op, DimShuffle):
            x = x.owner.inputs[0]
        return x

    def elem_inputs(x, want):
        """inputs of the Elemwise `want` that x is, under any DimShuffle layers, or None"""
        x = unshuffle(x)
        if x.owner is not None and scalar_op_name(x.owner) == want:
            return list(x.owner.inputs)
        return None

    def mul_leaves(x):
        """the factors of a product, by the graph's structure (constant factors are not folded together)"""
        x = unshuffle(x)
        if x.owner is not None and scalar_op_name(x.owner) == "mul":
            return [leaf for inp in x.owner.inputs for leaf in mul_leaves(inp)]
        return [x]

    def is_dot(x):
        x = unshuffle(x)
        return x.owner is not None and isinstance(x.owner.op, Dot)

    def omega_ls_of(d):
        """(omega [M][D], ls, the ls graph) of dot(square(omega), square(ls)), ls = ones(D) * ls as the covariance writes it"""
        d = unshuffle(d)
        a, b = (unshuffle(v) for v in d.owner.inputs)
        om = _const_value(a.owner.inputs[0]) if a.owner is not None and scalar_op_name(a.owner) == "sqr" else None
        if om is None:
            om2 = _const_value(a)
            om = None if om2 is None else np.sqrt(om2)
        if om is None or b.owner is None or scalar_op_name(b.owner) != "sqr":
            return None
        om = np.asarray(om, dtype=np.float64).reshape(len(om), -1)
        lsx = unshuffle(b.owner.inputs[0])
        c = _const_value(lsx)
        leaves = mul_leaves(lsx)
        if c is None and all(_const_value(leaf) is not None for leaf in leaves):  # ones(D) * ls, each factor constant
            c = np.prod([np.broadcast_to(_const_value(leaf), (om.shape[1],)) for leaf in leaves], axis=0)
        if c is not None:  # constant lengthscales: the D values
            return om, np.broadcast_to(np.asarray(c, dtype=np.float64).reshape(-1), (om.shape[1],)).copy(), lsx
        for leaf in leaves:
            if _const_value(leaf) is not None:
                continue  # the ones(D) the covariance multiplies ls by
            if leaf.owner is not None and scalar_op_name(leaf.owner) in ("truediv", "true_div", "reciprocal"):
                raise NotImplementedError("HSGP: a covariance given ls_inv is outside the closed set (give ls)")
            if leaf in name_of:
                if size_of[name_of[leaf]] not in (1, om.shape[1]):
                    raise NotImplementedError(f"HSGP: ls must be a scalar or one per input dimension ({HSGP_FORM})")
                return om, _ir.Ref(use(leaf)), lsx
            raise NotImplementedError(f"HSGP: ls must be constants, a scalar or a vector free RV ({HSGP_FORM})")
        return None

    def density_of(node, son):
        """(cov, omega, ls, ls graph) when the psd factor `node` is exp(-0.5 dot(...)) (ExpQuad) or
        power(c + dot(...), -(D + c) / 2) with c = 5 or 3 (Matern 5/2, 3/2), matched by structure; else None"""
        if son == "exp":
            ins = elem_inputs(node.inputs[0], "mul") or []
            dots = [v for v in ins if is_dot(v)]
            rest = [_const_value(v) for v in ins if not is_dot(v)]
            if len(dots) != 1 or len(rest) != 1 or rest[0] is None or rest[0].size != 1 or float(rest[0]) != -0.5:
                return None
            got = omega_ls_of(dots[0])
            return None if got is None else ("expquad",) + got
        if son == "pow":
            ins = elem_inputs(node.inputs[0], "add") or []
            dots = [v for v in ins if is_dot(v)]
            cs = [_const_value(v) for v in ins if not is_dot(v)]
            e = _const_value(node.inputs[1])
            if len(dots) != 1 or len(cs) != 1 or cs[0] is None or cs[0].size != 1 or e is None:
                return None
            got = omega_ls_of(dots[0])
            if got is None:
                return None
            c0, D = float(cs[0]), got[0].shape[1]
            cov = {5.0: "matern52", 3.0: "matern32"}.get(c0)
            if cov is None or float(e) != -(D + c0) / 2.0:
                raise NotImplementedError(f"HSGP: only the Matern 5/2 and 3/2 densities are in the closed set ({HSGP_FORM})")
            return (cov,) + got
        return None

    def spectral_of(psd, M):
        """ir.Spectral of sqrt_psd's argument psd (under psd[i:] when drop_first), else raise.  The factors are matched by
        the graph's structure before any constant is folded, so constant lengthscales keep their frequencies."""
        x, drop = unshuffle(psd), False
        if x.owner is not None and isinstance(x.owner.op, Subtensor) and not isinstance(x.owner.op, (AdvancedSubtensor, AdvancedSubtensor1)):
            x, drop = unshuffle(x.owner.inputs[0]), True
        if x.owner is not None and scalar_op_name(x.owner) == "add":
            raise NotImplementedError(f"HSGP: sums of kernels inside one term are outside the closed set (write one HSGP "
                                      f"per kernel and add them; {HSGP_FORM})")
        const, amp, found, prods = 1.0, None, [], []
        for leaf in mul_leaves(x):
            node = leaf.owner
            son = scalar_op_name(node) if node is not None else ""
            if node is not None and type(node.op).__name__.lower() == "prod":
                prods.append(unshuffle(node.inputs[0]))  # prod(ls): checked against the density's ls below
                continue
            got = density_of(node, son) if son in ("exp", "pow") else None
            if got is not None:
                found.append(got)
                continue
            c = _const_value(leaf)
            if c is not None:
                if c.size != 1:
                    raise NotImplementedError(f"HSGP: psd must be a scalar times the covariance's density ({HSGP_FORM})")
                const *= float(c.reshape(()))
                continue
            if leaf in name_of:
                raise NotImplementedError(f"HSGP: eta * cov with a random eta is outside the closed set (write eta**2 * cov; "
                                          f"{HSGP_FORM})")
            if son in ("sqr", "pow") and unshuffle(node.inputs[0]) in name_of:
                e = _const_value(node.inputs[1]) if son == "pow" else np.array(2.0)
                if e is None or float(e) != 2.0 or size_of[name_of[unshuffle(node.inputs[0])]] != 1:
                    raise NotImplementedError(f"HSGP: the amplitude must be eta**2 with eta a scalar free RV ({HSGP_FORM})")
                if amp is not None:
                    raise NotImplementedError(f"HSGP: products of kernels are outside the closed set ({HSGP_FORM})")
                amp = _ir.Ref(use(unshuffle(node.inputs[0])))
                continue
            if son == "exp":
                raise NotImplementedError(f"HSGP: exp(...) is not ExpQuad's density ({HSGP_FORM})")
            if son == "pow":
                raise NotImplementedError(f"HSGP: a power that is not a Matern density ({HSGP_FORM})")
            what = type(node.op).__name__ if node is not None else str(leaf)
            if son in ("ive", "iv", "i0", "i1", "besseli") or "bessel" in what.lower():
                raise NotImplementedError(f"HSGP: HSGPPeriodic is outside the closed set ({HSGP_FORM})")
            raise NotImplementedError(f"HSGP: {what} in the power spectral density is outside the closed set ({HSGP_FORM})")
        if len(found) != 1:
            raise NotImplementedError(("HSGP: products of kernels are outside the closed set" if found else
                                       "HSGP: no ExpQuad / Matern density in sqrt_psd") + f" ({HSGP_FORM})")
        cov, om, ls, lsx = found[0]
        if len(prods) != 1 or prods[0] is not lsx:
            raise NotImplementedError(f"HSGP: the density must hold prod(ls) of the ls in its exponent once "
                                      f"({HSGP_FORM})")
        if drop:
            om = om[1:]
        if om.shape[0] != M:
            raise NotImplementedError(f"HSGP: phi has {M} columns but psd {om.shape[0]} frequencies ({HSGP_FORM})")
        scale2 = const / np.exp(_ir.spectral_log_const(cov, om.shape[1])[0])
        if amp is not None and abs(scale2 - 1.0) > 1e-12:
            raise NotImplementedError(f"HSGP: eta**2 times a further constant is outside the closed set ({HSGP_FORM})")
        return _ir.Spectral(cov, om, ls, amp if amp is not None else float(np.sqrt(scale2)))

    def hsgp_of(b, Phi):
        """(z, ir.Spectral) of b = z * sqrt(psd) (either order), z a free RV of Phi's width, or (z, s) with s the M
        constants of an already folded sqrt_psd; else None"""
        ins = elem_inputs(b, "mul")
        if ins is None or len(ins) != 2:
            return None
        for z, sq in (ins, ins[::-1]):
            z = unshuffle(z)
            if z not in name_of or size_of[name_of[z]] != Phi.shape[1]:
                continue
            root = elem_inputs(sq, "sqrt")
            if root is not None:
                return z, spectral_of(root[0], Phi.shape[1])
            s = _const_value(sq)
            if s is not None and s.shape == (Phi.shape[1],):
                return z, np.asarray(s, dtype=np.float64)
        return None
        for z, sq in (ins, ins[::-1]):
            z, root = unshuffle(z), inputs_of(sq, "sqrt")
            if z in name_of and size_of[name_of[z]] == Phi.shape[1] and root is not None:
                return z, spectral_of(root[0], Phi.shape[1])
        return None

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
        if op == "dirichlet":  # multivariate.py:557-585; its value variable is the simplex of K - 1 coordinates
            a = _const_value(ps[0])
            if a is None:
                raise NotImplementedError(f"{rv.name}: a pm.Dirichlet with a random a is outside the closed set (a is a "
                                          "constant)")
            priors.append(_ir.Prior("dirichlet", vn, (np.asarray(a, dtype=np.float64),)))
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
            sq = unshuffle(ps[i])
            if i == scale and c is None and sq.owner is not None and scalar_op_name(sq.owner) == "sqrt":
                raise NotImplementedError(f"{rv.name}: the centred HSGP parametrisation (a Normal prior whose sigma is "
                                          "sqrt_psd, a vector of random scales) is outside the closed set: use "
                                          "parametrization='noncentered'")
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

    def graph_nodes(x):
        """every variable with an owner in the graph under x"""
        out, seen, stack = [], set(), [x]
        while stack:
            v = stack.pop()
            if v.owner is None or id(v) in seen:
                continue
            seen.add(id(v))
            out.append(v)
            stack.extend(v.owner.inputs)
        return out

    def cutpoints_of(x):
        """a vector free RV (-> Ref) or a constant 1-D array of cutpoints under DimShuffle layers, else None"""
        while x.owner is not None and isinstance(x.owner.op, DimShuffle):
            x = x.owner.inputs[0]
        if x in name_of:
            return _ir.Ref(use(x))
        c = _const_value(x)
        return np.asarray(c, dtype=np.float64) if c is not None and c.ndim == 1 else None

    def ordinal_of(p):
        """(dist, eta, cutpoints, sigma) of a Categorical p built by OrderedLogistic.compute_p (discrete.py:1312-1326:
        differences of a concatenation around sigmoid(cutpoints - eta[:, None])) or OrderedProbit.compute_p (:1416-1432:
        exp of a concatenation of normal_lccdf / log_diff_normal_cdf / normal_lcdf of eta[:, None] - cutpoints, each
        standardising as (x - 0) / sigma, dist_math.py:126-182), else None"""
        while p.owner is not None and _is_copy(p.owner):  # the {name}_probs Deterministic (compute_p=True)
            p = p.owner.inputs[0]
        if p.owner is None:
            return None
        nodes = graph_nodes(p)
        ops = {scalar_op_name(v.owner) for v in nodes}
        top = scalar_op_name(p.owner)
        if top == "sub" and "sigmoid" in ops:
            for v in nodes:
                if scalar_op_name(v.owner) == "sigmoid":
                    inner = v.owner.inputs[0]
                    if inner.owner is not None and scalar_op_name(inner.owner) == "sub":
                        c = cutpoints_of(inner.owner.inputs[0])
                        if c is not None:
                            return "ordered_logistic", inner.owner.inputs[1], c, None
            return None
        if top != "exp" or not ops & {"erfc", "erfcx", "erf"}:
            return None
        probits = None
        for v in nodes:
            if scalar_op_name(v.owner) == "sub":
                c = cutpoints_of(v.owner.inputs[1])
                if c is not None and (isinstance(c, _ir.Ref) or c.size >= 1):
                    probits = v
                    break
        if probits is None:
            return None
        sigmas = []
        for v in nodes:  # (x - mu) / sigma with x a slice of the probits
            if scalar_op_name(v.owner) in ("truediv", "true_div"):
                num, den = v.owner.inputs
                if num.owner is not None and scalar_op_name(num.owner) == "sub" and \
                        any(w is probits for w in graph_nodes(num.owner.inputs[0])):
                    sigmas.append(den)
        if not sigmas:
            return None
        s = [param(d.owner.inputs[0] if d.owner is not None and isinstance(d.owner.op, DimShuffle) else d, "sigma")
             for d in sigmas]
        if any(t != s[0] for t in s):
            return None
        return "ordered_probit", probits.owner.inputs[0], cutpoints_of(probits.owner.inputs[1]), s[0]

    def family_of(op, ps, name, N):
        """(dist, eta, parameter slot) of a count / positive family RV (op, its dist params ps): pm.Poisson(mu=exp(eta)),
        pm.Binomial(n, logit_p=eta), pm.NegativeBinomial(mu=exp(eta), alpha), pm.Gamma(alpha, beta=alpha / exp(eta));
        observed likelihoods and the components of zero-inflated / hurdle mixtures share it."""
        if op == "poisson":
            eta = strip(ps[0], "exp")
            if eta is None:
                raise NotImplementedError(f"{name}: write the rate as pm.math.exp(linear predictor)")
            return "poisson_log", eta, {}
        if op == "binomial":  # RV parameters (n, p); logit_p= and p=invlogit(eta) both give p = sigmoid(eta)
            form = "pm.Binomial(n=trials, logit_p=linear predictor) with constant trials"
            nt = _const_value(ps[0])
            eta = inputs_of(ps[1], "sigmoid")
            if nt is None or eta is None:
                raise NotImplementedError(f"{name}: write the likelihood as {form}")
            trials = float(nt.reshape(())) if nt.size == 1 else np.ravel(np.broadcast_to(nt, (N,))).astype(np.float64)
            return "binomial_logit", eta[0], {"trials": trials}
        if op in ("negbinomial", "nbinom"):  # RV parameters (n = alpha, p = alpha / (mu + alpha)), discrete.py:700-723
            form = "pm.NegativeBinomial(mu=pm.math.exp(linear predictor), alpha=constant or scalar free RV)"
            try:
                alpha = param(ps[0], name + ".alpha")
            except NotImplementedError:
                raise NotImplementedError(f"{name}: write the likelihood as {form}") from None
            div, eta = inputs_of(ps[1], "truediv"), None
            den = inputs_of(div[1], "add") if div is not None and same_param(div[0], alpha) else None
            if den is not None and len(den) == 2:
                for mu_, a_ in (den, den[::-1]):
                    e = inputs_of(mu_, "exp")
                    if e is not None and same_param(a_, alpha):
                        eta = e[0]
                        break
            if eta is None:
                raise NotImplementedError(f"{name}: write the likelihood as {form}")
            return "negative_binomial_log", eta, {"alpha": alpha}
        # op == "gamma": RV parameters (alpha, scale = reciprocal(beta)), continuous.py:2478-2510
        form = ("pm.Gamma(alpha=a, beta=a / pm.math.exp(linear predictor)) or beta=a * pm.math.exp(-linear predictor), "
                "a a constant or scalar free RV")
        try:
            alpha = param(ps[0], name + ".alpha")
        except NotImplementedError:
            raise NotImplementedError(f"{name}: write the likelihood as {form}") from None
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
            raise NotImplementedError(f"{name}: write the likelihood as {form}")
        return "gamma_log", eta, {"alpha": alpha}

    def stack_of(w):
        """the entries of a stack / join / make_vector of scalars or vectors along the last axis, under DimShuffle layers"""
        while w.owner is not None and isinstance(w.owner.op, DimShuffle):
            w = w.owner.inputs[0]
        if w.owner is None or type(w.owner.op).__name__ not in ("Join", "MakeVector", "Stack"):
            return None
        ins = list(w.owner.inputs)
        if type(w.owner.op).__name__ == "Join":
            ins = ins[1:]  # the axis
        out = []
        for x in ins:
            while x.owner is not None and isinstance(x.owner.op, DimShuffle):
                x = x.owner.inputs[0]
            out.append(x)
        return out

    def psi_of(w, name, N):
        """psi of mixture weights stack([1 - psi, psi], axis=-1): a constant, a scalar free RV (-> Ref), or
        invlogit / sigmoid of a linear predictor (-> Linear, the logit of psi)"""
        form = ("the weights of a zero-inflated / hurdle mixture are stack([1 - psi, psi]) with psi a constant, a scalar "
                "free RV or pm.math.invlogit(linear predictor)")
        ent = stack_of(w)
        if ent is None or len(ent) != 2:
            raise NotImplementedError(f"{name}: {form}")
        one_minus, p = ent
        sub = inputs_of(one_minus, "sub")
        if sub is None or len(sub) != 2 or _const_value(sub[0]) is None or np.any(_const_value(sub[0]) != 1.0):
            raise NotImplementedError(f"{name}: {form}")
        q = sub[1]
        while q.owner is not None and isinstance(q.owner.op, DimShuffle):
            q = q.owner.inputs[0]
        if q is not p:
            raise NotImplementedError(f"{name}: {form}")
        z = inputs_of(p, "sigmoid")
        if z is not None:
            return _ir.Linear(make_terms(z[0], N))
        if p in name_of and size_of[name_of[p]] != 1:
            raise NotImplementedError(f"{name}: a vector psi variable is outside the closed set (psi is a constant, a "
                                      "scalar free RV or pm.math.invlogit(linear predictor))")
        c = _const_value(p)
        if c is not None and c.size != 1:
            raise NotImplementedError(f"{name}: a per-observation constant psi is outside the closed set (psi is a "
                                      "constant, a scalar free RV or pm.math.invlogit(linear predictor))")
        try:
            return param(p, name + ".psi")
        except NotImplementedError:
            raise NotImplementedError(f"{name}: {form}") from None

    def zero_inflated_of(rv, ps, N):
        """(dist, eta, parameter slot, psi) of pm.ZeroInflated* (a Mixture of [DiracDelta(0), f], mixture.py:560-574) or
        pm.Hurdle* (a _Hurdle of [DiracDelta(0), Truncated(f, lower=1) | Gamma], :812-844)"""
        hurdle = "hurdle" in _op_name(rv)
        w, comps = ps[0], ps[1:]
        zero = comps[0] if comps else None
        if len(comps) != 2 or zero.owner is None or _op_name(zero) != "diracdelta" or \
                _const_value(_dist_params(zero)[0]) is None or np.any(_const_value(_dist_params(zero)[0]) != 0):
            raise NotImplementedError(f"{rv.name}: a list-of-components pm.Mixture / pm.NormalMixture is outside the closed "
                                      "set (write the K components as one batched distribution: pm.NormalMixture(w, mu, "
                                      "sigma) or pm.Mixture(w, pm.Poisson.dist(lam, shape=K)); the other two-component "
                                      "mixtures are the zero-inflated Poisson, Binomial and NegativeBinomial)")
        comp = comps[1]
        cop = _op_name(comp)
        if hurdle and cop == "lognormal":
            raise NotImplementedError(f"{rv.name}: pm.HurdleLogNormal is outside the closed set (the hurdle likelihoods "
                                      "are HurdlePoisson, HurdleNegativeBinomial and HurdleGamma)")
        cps = _dist_params(comp)
        truncated = cop == "truncated"
        if hurdle and truncated:  # Truncated(f, lower=1): f's own parameters, then lower and upper
            cop = _op_class_name(comp.owner.op.base_rv_op)
            lo, hi = _const_value(cps[-2]), _const_value(cps[-1])
            if lo is None or hi is None or np.any(lo != 1) or np.any(hi != np.inf):
                raise NotImplementedError(f"{rv.name}: a hurdle's count component is Truncated(f, lower=1)")
            cps = cps[: -2][-({"poisson": 1}.get(cop, 2)):]
        # a hurdle's count component is Truncated(f, lower=1), its Gamma component the Gamma itself
        ok = (truncated and cop in ("poisson", "negbinomial", "nbinom")) or (not truncated and cop == "gamma") if hurdle else \
            cop in ("poisson", "binomial", "negbinomial", "nbinom")
        if not ok:
            what = "pm.HurdlePoisson / HurdleNegativeBinomial / HurdleGamma" if hurdle else \
                "pm.ZeroInflatedPoisson / ZeroInflatedBinomial / ZeroInflatedNegativeBinomial"
            raise NotImplementedError(f"{rv.name}: a mixture with a {type(comp.owner.op).__name__} component is outside "
                                      f"the closed set (only {what})")
        fam, eta, slot = family_of(cop, cps, rv.name, N)
        dist = next(d for d, f in _ir.ZI_FAMILY.items() if f == fam and d.startswith("hurdle" if hurdle else "zero"))
        return dist, eta, slot, psi_of(w, rv.name, N)

    def peel(x):
        while x.owner is not None and isinstance(x.owner.op, DimShuffle):
            x = x.owner.inputs[0]
        return x

    def mixture_of(rv, ps, N):
        """Likelihood arguments of a Mixture of ONE batched component (mixture.py:469-494, :529-546): pm.NormalMixture(w,
        mu, sigma) -> normal_mixture, pm.Mixture(w, pm.Poisson.dist(lam, shape=K)) -> poisson_mixture, seen through the
        DimShuffle / broadcast layers of PyMC's resizing to (N, K)"""
        name, comp = rv.name, ps[1]
        cop = _op_name(comp) if comp.owner is not None else ""
        if cop not in ("normal", "poisson"):
            what = type(comp.owner.op).__name__ if comp.owner is not None else str(comp)
            raise NotImplementedError(f"{name}: a mixture of {what} components is outside the closed set (only Normal "
                                      "and Poisson components)")
        # the weights: a free pm.Dirichlet (simplex) or a constant K-vector
        wv = peel(ps[0])
        wform = "the weights of a mixture are a free pm.Dirichlet or a constant K-vector"
        if wv in name_of:
            if name_of[wv] not in simplex:
                raise NotImplementedError(f"{name}: {wform}")
            weights, K = _ir.Ref(name_of[wv]), size_of[name_of[wv]] + 1
        else:
            c = _const_value(wv)
            if c is None:
                raise NotImplementedError(f"{name}: {wform}")
            c = np.asarray(c, dtype=np.float64)
            if c.ndim > 1 and not np.all(c.reshape(-1, c.shape[-1]) == c.reshape(-1, c.shape[-1])[0]):
                raise NotImplementedError(f"{name}: per-observation weights are outside the closed set ({wform})")
            weights = c.reshape(-1, c.shape[-1])[0] if c.ndim else c
            K = int(np.size(weights))

        def per_component(x, what):
            """a free RV of size K (or 1 where allowed: -> Ref) or a constant of 1 or K values, else None"""
            x = peel(x)
            if x in name_of:
                vn = name_of[x]
                if vn in simplex:
                    raise NotImplementedError(f"{x.name}: {_ir.SIMPLEX_USE} (pm.NormalMixture / pm.Mixture w)")
                if size_of[vn] not in (1, K):
                    raise NotImplementedError(f"{name}: a per-observation {what} is outside the closed set (one per "
                                              "component)")
                return _ir.Ref(vn), size_of[vn]
            c = _const_value(x)
            if c is None:
                return None
            c = np.asarray(c, dtype=np.float64)
            if c.ndim > 1 and not np.all(c.reshape(-1, c.shape[-1]) == c.reshape(-1, c.shape[-1])[0]):
                raise NotImplementedError(f"{name}: a per-observation {what} is outside the closed set (one per component)")
            v = c.reshape(-1, c.shape[-1])[0] if c.ndim else c.reshape(1)
            return (float(v[0]) if v.size == 1 and what == "sigma" else v), v.size

        def split(x, join, what, mark):
            """(component, eta or None) of x = component, or x = join(eta-part, component) where mark(eta-part) gives eta"""
            ins = inputs_of(x, join)
            if ins is not None and len(ins) == 2:
                for a, b in ((ins[0], ins[1]), (ins[1], ins[0])):  # the component is the part with K values
                    eta = mark(a)
                    try:
                        got = per_component(b, what) if eta is not None else None
                    except NotImplementedError:
                        got = None
                    if got is not None and got[1] == K:
                        return got[0], eta
            got = per_component(x, what)
            return (got[0], None) if got is not None else (None, None)

        cps = _dist_params(comp)
        if cop == "normal":
            form = ("pm.NormalMixture(w, mu, sigma) with mu a K-vector free RV or constant, optionally "
                    "linear_predictor[:, None] + mu, and sigma a constant, a scalar free RV or a K-vector free RV")
            mu, eta = split(cps[0], "add", "mu", peel)
            if mu is None:
                raise NotImplementedError(f"{name}: {form}")
            s = peel(cps[1])
            if s.owner is not None and scalar_op_name(s.owner) in ("pow", "reciprocal", "sqrt", "invsqrt", "truediv"):
                raise NotImplementedError(f"{name}: pm.NormalMixture(tau=...) is outside the closed set (give sigma)")
            got = per_component(s, "sigma")
            if got is None:
                raise NotImplementedError(f"{name}: {form}")
            return "normal_mixture", eta, dict(weights=weights, components=mu, sigma=got[0])
        form = ("pm.Mixture(w, pm.Poisson.dist(lam, shape=K)) with lam a K-vector free RV or constant, optionally "
                "pm.math.exp(linear_predictor)[:, None] * lam")
        lam, eta = split(cps[0], "mul", "lam", lambda a: (inputs_of(a, "exp") or [None])[0])
        if lam is None:
            raise NotImplementedError(f"{name}: {form}")
        return "poisson_mixture", eta, dict(weights=weights, components=lam)

    def survival_of(op, ps, name, sigma_of):
        """(family, eta, parameter slot) of a survival RV (op, its dist params ps): pm.Weibull(alpha, beta=exp(eta)),
        pm.Exponential(scale=exp(eta)) or (lam=exp(-eta)) -- the Weibull with alpha = 1 -- or pm.LogNormal(eta, sigma)"""
        if op in ("weibullbeta", "weibull"):  # WeibullBetaRV: (alpha, beta), continuous.py:2717-2737
            form = "pm.Weibull(alpha, beta=pm.math.exp(linear predictor)) with alpha a constant or a scalar free RV"
            a = ps[0]
            while a.owner is not None and isinstance(a.owner.op, DimShuffle):
                a = a.owner.inputs[0]
            c = _const_value(a)
            if (a in name_of and size_of[name_of[a]] != 1) or (a not in name_of and c is not None and c.size != 1):
                raise NotImplementedError(f"{name}: a per-observation or vector Weibull alpha is outside the closed set "
                                          f"({form})")
            try:
                alpha = param(a, name + ".alpha")
            except NotImplementedError:
                raise NotImplementedError(f"{name}: a Weibull alpha that is an expression of random variables is outside "
                                          f"the closed set ({form})") from None
            e = inputs_of(ps[1], "exp")
            if e is None:
                raise NotImplementedError(f"{name}: write the likelihood as {form}")
            return "weibull_log", e[0], {"alpha": alpha}
        if op == "exponential":  # ExponentialRV: (scale,), scale = reciprocal(lam), continuous.py:1461-1471
            form = ("pm.Exponential(scale=pm.math.exp(linear predictor)) or "
                    "pm.Exponential(lam=pm.math.exp(-linear predictor))")
            e, eta = inputs_of(ps[0], "exp"), None
            if e is not None:
                eta = e[0]
            else:
                r = inputs_of(ps[0], "reciprocal")
                e = inputs_of(r[0], "exp") if r is not None else None
                ng = inputs_of(e[0], "neg") if e is not None else None
                eta = ng[0] if ng is not None else None
            if eta is None:
                raise NotImplementedError(f"{name}: write the likelihood as {form}")
            return "weibull_log", eta, {"alpha": 1.0}
        return "lognormal", ps[0], {"sigma": sigma_of(ps[1])}  # LogNormalRV: (mu, sigma)

    def beta_of(op, ps, name, N):
        """(dist, eta, slots) of pm.Beta / pm.BetaBinomial whose alpha = mu * phi and beta = (1 - mu) * phi (the factors of
        each product in either order), mu = invlogit(eta): BetaRV (alpha, beta), the graph get_alpha_beta builds for
        Beta(mu, nu) too (continuous.py:1238-1240); BetaBinomialRV (n, alpha, beta), discrete.py:178-262"""
        bb = op == "betabinomial"
        form = ("pm.BetaBinomial(alpha=mu * phi, beta=(1 - mu) * phi, n=trials) with constant trials" if bb else
                "pm.Beta(mu=mu, nu=phi) or pm.Beta(alpha=mu * phi, beta=(1 - mu) * phi)") + \
            ", mu = pm.math.invlogit(linear predictor) and phi a constant or a scalar free RV"
        a_, b_ = ps[-2], ps[-1]
        slots = {}
        if bb:
            nt = _const_value(ps[0])
            if nt is None:
                raise NotImplementedError(f"{name}: random trials are outside the closed set ({form})")
            slots["trials"] = float(nt.reshape(())) if nt.size == 1 else np.ravel(np.broadcast_to(nt, (N,))).astype(np.float64)
        if _const_value(a_) is not None and _const_value(b_) is not None:
            raise NotImplementedError(f"{name}: constant alpha and beta with no predictor are outside the closed set (write "
                                      f"{form})")
        ins = inputs_of(a_, "mul")
        if ins is None or len(ins) != 2:
            raise NotImplementedError(f"{name}: write the likelihood as {form}")
        mu = next(((m_, p_) for m_, p_ in (ins, ins[::-1]) if inputs_of(m_, "sigmoid") is not None), None)
        if mu is None:
            raise NotImplementedError(f"{name}: a mean other than invlogit of a linear predictor is outside the closed set "
                                      f"({form})")
        mu, p_ = peel(mu[0]), peel(mu[1])
        if p_.owner is not None and p_ not in name_of and \
                {scalar_op_name(v.owner) for v in graph_nodes(p_)} & {"pow", "sqr", "sqrt"}:
            raise NotImplementedError(f"{name}: pm.Beta(mu, sigma), the kappa form, is outside the closed set (write {form})")
        c = _const_value(p_)
        if (p_ in name_of and size_of[name_of[p_]] != 1) or (p_ not in name_of and c is not None and c.size != 1):
            raise NotImplementedError(f"{name}: a per-observation or vector phi is outside the closed set ({form})")
        try:
            phi = param(p_, name + ".phi")
        except NotImplementedError:
            raise NotImplementedError(f"{name}: a phi that is an expression of random variables is outside the closed set "
                                      f"({form})") from None
        ok = False
        ins = inputs_of(b_, "mul")
        for one_minus, q_ in (ins, ins[::-1]) if ins is not None and len(ins) == 2 else ():
            sub = inputs_of(one_minus, "sub")
            one = _const_value(sub[0]) if sub is not None and len(sub) == 2 else None
            if one is not None and np.all(one == 1.0) and peel(sub[1]) is mu and same_param(q_, phi):
                ok = True
        if not ok:
            raise NotImplementedError(f"{name}: write the likelihood as {form} (beta must be (1 - mu) * phi with the mu "
                                      "and phi of alpha)")
        return ("beta_binomial_logit" if bb else "beta_logit"), inputs_of(mu, "sigmoid")[0], dict(slots, phi=phi)

    survival_ops = ("weibullbeta", "weibull", "exponential", "lognormal")
    probs_of = {}  # id of a {name}_probs Deterministic's expression -> the ordinal likelihood's name
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
        elif op in ("poisson", "binomial", "negbinomial", "nbinom", "gamma"):
            dist, eta, slot = family_of(op, ps, rv.name, N)
            liks.append(_ir.Likelihood(dist, y, make_terms(eta, N), name=rv.name, **slot))
        elif op == "mixture" and len(ps) == 2:  # pm.NormalMixture / pm.Mixture of one batched component
            dist, eta, kw = mixture_of(rv, ps, N)
            liks.append(_ir.Likelihood(dist, y, [] if eta is None else make_terms(eta, N), name=rv.name, **kw))
        elif op in ("mixture", "_hurdle", "hurdle"):  # pm.ZeroInflated* / pm.Hurdle*
            dist, eta, slot, psi = zero_inflated_of(rv, ps, N)
            liks.append(_ir.Likelihood(dist, y, make_terms(eta, N), name=rv.name, psi=psi, **slot))
        elif op in ("beta", "betabinomial"):
            dist, eta, slot = beta_of(op, ps, rv.name, N)
            liks.append(_ir.Likelihood(dist, y, make_terms(eta, N), name=rv.name, **slot))
        elif op in survival_ops:
            dist, eta, slot = survival_of(op, ps, rv.name, sigma_of)
            liks.append(_ir.Likelihood(dist, y, make_terms(eta, N), name=rv.name, **slot))
        elif op in ("censored", "truncatednormal", "truncated"):
            # CensoredRV: dist params (base, lower, upper) (censored.py:45-76); TruncatedNormalRV: (mu, sigma, lower, upper)
            # (continuous.py:558-583), which pm.Truncated of a Normal also becomes (truncated.py:499-505); TruncatedRV
            # (truncated.py:53-130): the base RV's own inputs followed by lower and upper, its op in base_rv_op
            def bound(x, open_value):
                v = _const_value(x)
                if v is None:
                    raise NotImplementedError(f"{rv.name}: censoring / truncation bounds must be constants (random bounds are "
                                              "outside the closed set)")
                v = np.asarray(v, dtype=np.float64)
                if v.size == 1:
                    return None if float(v.reshape(())) == open_value else float(v.reshape(()))
                return np.ravel(np.broadcast_to(v, (N,))).astype(np.float64)

            if op == "truncated":
                base_op = getattr(rv.owner.op, "base_rv_op", None)
                what = type(base_op).__name__ if base_op is not None else type(rv.owner.op).__name__
                bop = _op_class_name(base_op) if base_op is not None else ""
                if bop not in survival_ops:
                    raise NotImplementedError(f"{rv.name}: pm.Truncated of {what} is outside the closed set (only a "
                                              "Normal, Weibull, Exponential or LogNormal base distribution can be truncated)")
                lo, hi = ps[-2], ps[-1]
                fam, eta, slot = survival_of(bop, ps[:-2][-(1 if bop == "exponential" else 2):], rv.name, sigma_of)
                liks.append(_ir.Likelihood(f"truncated_{fam}", y, make_terms(eta, N), lower=bound(lo, -np.inf),
                                           upper=bound(hi, np.inf), name=rv.name, **slot))
                continue
            if op == "truncatednormal":
                mu, s, lo, hi = ps[:4]
            else:
                base, lo, hi = ps[:3]
                bop = _op_name(base) if base.owner is not None else ""
                if bop == "truncated":
                    raise NotImplementedError(f"{rv.name}: pm.Censored of a pm.Truncated distribution is outside the closed "
                                              "set (censor or truncate, not both)")
                if bop in survival_ops:
                    fam, eta, slot = survival_of(bop, _dist_params(base), rv.name, sigma_of)
                    liks.append(_ir.Likelihood(f"censored_{fam}", y, make_terms(eta, N), lower=bound(lo, -np.inf),
                                               upper=bound(hi, np.inf), name=rv.name, **slot))
                    continue
                if bop != "normal":
                    what = type(base.owner.op).__name__ if base.owner is not None else str(base)
                    raise NotImplementedError(f"{rv.name}: pm.Censored of {what} is outside the closed set (only a Normal, "
                                              "Weibull, Exponential or LogNormal base distribution can be censored)")
                mu, s = _dist_params(base)[:2]
            dist = "censored_normal" if op == "censored" else "truncated_normal"
            liks.append(_ir.Likelihood(dist, y, make_terms(mu, N), sigma=sigma_of(s), lower=bound(lo, -np.inf),
                                       upper=bound(hi, np.inf), name=rv.name))
        elif op == "categorical":  # pm.OrderedLogistic / pm.OrderedProbit build Categorical(p = compute_p(eta, cutpoints))
            form = ("pm.OrderedLogistic(eta, cutpoints) or pm.OrderedProbit(eta, cutpoints, sigma): a Categorical with a "
                    "free p, logit_p / softmax, or a p of another form is outside the closed set")
            found = ordinal_of(ps[0])
            if found is None:
                raise NotImplementedError(f"{rv.name}: Categorical: only {form}")
            dist, eta, cut, s = found
            if isinstance(cut, _ir.Ref) and size_of[cut.var] > 1 and \
                    next(v for v in vars_ if v.name == cut.var).transform not in _ir.ORDERED_TRANSFORMS:
                raise NotImplementedError(f"{rv.name}: the cutpoints {cut.var} need transform=pm.distributions.transforms."
                                          "ordered (unordered vector cutpoints)")
            liks.append(_ir.Likelihood(dist, y, make_terms(eta, N), sigma=s, cutpoints=cut, name=rv.name))
            probs_of[id(ps[0])] = rv.name
        else:
            raise NotImplementedError(f"{rv.name}: likelihood {type(rv.owner.op).__name__} is outside the closed set "
                                      f"{sorted(_ir.LIK_DISTS)}")
    # ---- pm.Deterministic: recorded in the posterior, never part of logp -------------------------------------------------
    dets = []
    for dv in getattr(model, "deterministics", []) or []:
        if id(dv) in probs_of:  # {name}_probs of an ordinal likelihood: evaluated from its own factor
            L = next(L for L in liks if L.name == probs_of[id(dv)])
            K = (size_of[L.cutpoints.var] if isinstance(L.cutpoints, _ir.Ref) else len(L.cutpoints)) + 1
            dets.append(_ir.Deterministic(dv.name, len(L.y) * K, [], probs_of=L.name))
            continue
        size = _static_size(dv)
        if size is None:
            raise NotImplementedError(f"{dv.name}: the size of this Deterministic is not known statically")
        expr = dv
        if expr.owner is not None and _is_copy(expr.owner):
            expr = expr.owner.inputs[0]  # pm.Deterministic wraps its expression in a named copy
        dets.append(_ir.Deterministic(dv.name, size, make_terms(expr, size)))
    out = _ir.ModelIR(vars_, priors, liks, ar1, name=getattr(model, "name", "") or "pymc_model", deterministics=dets)
    out.validate()
    return out
