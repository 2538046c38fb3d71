"""Model specifications for the sampling engine (the hand-lowered stand-in for a PyTensor graph).

In the reference a model reaches the sampler as ONE compiled callable ``q[n] -> (logp, dlogp[n])``
built by ``Model.logp_dlogp_function`` (pymc/model/core.py:464-529) over the raveled, transformed
value variables in registration order (pymc/pytensorf.py:575-595, pymc/blocking.py:68-75).  A
``ModelSpec`` carries exactly what that callable closes over: the ordered value-variable layout
(names as PyMC would name them, ``"{rv}_{transform}__"``, pymc/model/core.py:2141-2153), the observed
data, and a ``kind`` that selects the hand-written device function fusing the joint log-density
and its reverse-mode gradient (pymc_b200/csrc/models.cuh).

The five kinds are the five BASELINE.json configs; their synthetic data follows SURVEY.md 8(d)
(the reference ships no data: radon.csv is fetched over the network, pymc/data.py:63).
"""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np

# kind ids shared with include/b200nuts.h (B200_MODEL_*)
KIND_STD_NORMAL = 0
KIND_EIGHT_SCHOOLS = 1
KIND_RADON = 2
KIND_LOGISTIC = 3
KIND_STOCHVOL = 4
KIND_MVGAUSS = 5
KIND_IR = 6  # any ModelIR on the generic device function (pymc_b200.ir)

KIND_NAMES = {
    KIND_STD_NORMAL: "std_normal",
    KIND_EIGHT_SCHOOLS: "eight_schools",
    KIND_RADON: "radon",
    KIND_LOGISTIC: "logistic",
    KIND_STOCHVOL: "stochvol",
    KIND_MVGAUSS: "mvgauss",
    KIND_IR: "ir",
}


@dataclass
class VarInfo:
    """One value variable inside the raveled vector q."""

    name: str  # value-variable name, e.g. "tau_log__"
    rv_name: str  # random-variable name, e.g. "tau"
    offset: int
    size: int
    transform: str | None = None  # None | "log" | "interval" | "ordered" | "ordered_positive" | "simplex"
    bounds: tuple[float, float] | None = None  # for "interval"


@dataclass
class ModelSpec:
    kind: int
    n: int
    vars: list[VarInfo]
    data: dict[str, np.ndarray] = field(default_factory=dict)
    meta: dict = field(default_factory=dict)

    @property
    def name(self) -> str:
        return KIND_NAMES[self.kind]

    @property
    def var_sizes(self) -> dict[str, int]:
        return {v.name: v.size for v in self.vars}

    def split(self, q: np.ndarray) -> dict[str, np.ndarray]:
        """Unravel ``q[..., n]`` into value variables (DictToArrayBijection.rmap, blocking.py:78-103)."""
        return {v.name: q[..., v.offset : v.offset + v.size] for v in self.vars}

    def constrain(self, q: np.ndarray) -> dict[str, np.ndarray]:
        """Unconstrained draws -> named constrained RVs (what NDArray.record evaluates per draw,
        pymc/backends/ndarray.py:108; transforms per pymc/logprob/transforms.py:880-891, :1026-1045)."""
        out = {}
        for v in self.vars:
            x = q[..., v.offset : v.offset + v.size]
            if v.transform == "log":
                x = np.exp(x)
            elif v.transform == "interval":
                a, b = v.bounds
                s = 1.0 / (1.0 + np.exp(-x))
                x = s * b + (1.0 - s) * a
            elif v.transform in ("ordered", "ordered_positive"):  # Ordered.backward, transforms.py:96-106
                d = np.exp(x)
                if v.transform == "ordered":
                    d[..., 0] = x[..., 0]
                x = np.cumsum(d, axis=-1)
            elif v.transform == "simplex":  # SimplexTransform.backward, transforms.py:1101-1105: size + 1 weights
                from .ir import simplex_backward

                out[v.rv_name] = simplex_backward(x)
                continue
            if v.size == 1:
                x = x[..., 0]
            out[v.rv_name] = x
        return out

    def split_rv(self, x: np.ndarray) -> dict[str, np.ndarray]:
        """Already-constrained draws ``x[..., n]`` (recorded that way by the kernel) -> named RVs."""
        out = {}
        for v in self.vars:
            a = x[..., v.offset : v.offset + v.size]
            out[v.rv_name] = a[..., 0] if v.size == 1 else a
        return out

    def initial_point(self) -> np.ndarray:
        """The model's default initial point in unconstrained space (support point of every prior,
        transformed; pymc/initial_point.py).  All five configs have support points that map to 0
        except where noted in ``meta['initial_point']``."""
        ip = self.meta.get("initial_point")
        return np.zeros(self.n) if ip is None else np.asarray(ip, dtype=np.float64).copy()


def _layout(entries) -> tuple[list[VarInfo], int]:
    out, off = [], 0
    for name, rv, size, tr, bounds in entries:
        out.append(VarInfo(name, rv, off, size, tr, bounds))
        off += size
    return out, off


# ------------------------------------------------------------------------------------------------
# config 0 (tests only): iid standard normal, the "trivial logp" of BASELINE.md section 2
# ------------------------------------------------------------------------------------------------
def std_normal(n: int) -> ModelSpec:
    vars_, n_ = _layout([("x", "x", n, None, None)])
    return ModelSpec(KIND_STD_NORMAL, n_, vars_)


# ------------------------------------------------------------------------------------------------
# config 1: Eight Schools, non-centred
# ------------------------------------------------------------------------------------------------
EIGHT_SCHOOLS_Y = np.array([28.0, 8.0, -3.0, 7.0, -1.0, 1.0, 18.0, 12.0])
EIGHT_SCHOOLS_SIGMA = np.array([15.0, 10.0, 16.0, 11.0, 9.0, 11.0, 10.0, 18.0])


def eight_schools() -> ModelSpec:
    """mu~Normal(0,5); tau~HalfCauchy(5) [log]; theta_t~Normal(0,1,8); y~Normal(mu+tau*theta_t, sigma)."""
    vars_, n = _layout(
        [
            ("mu", "mu", 1, None, None),
            ("tau_log__", "tau", 1, "log", None),
            ("theta_t", "theta_t", 8, None, None),
        ]
    )
    # HalfCauchy(5) support point is beta=5 -> log 5 on the unconstrained scale
    ip = np.zeros(n)
    ip[1] = np.log(5.0)
    return ModelSpec(
        KIND_EIGHT_SCHOOLS,
        n,
        vars_,
        data={"y": EIGHT_SCHOOLS_Y.copy(), "sigma": EIGHT_SCHOOLS_SIGMA.copy()},
        meta={"initial_point": ip},
    )


# ------------------------------------------------------------------------------------------------
# config 2: Radon hierarchical regression (benchmarks/benchmarks/benchmarks.py:26-46)
# ------------------------------------------------------------------------------------------------
def radon_data(n_obs: int = 919, n_counties: int = 85, seed: int = 123):
    """Synthetic radon-shaped data (SURVEY 8d): county sizes ~ multinomial with every county >= 1."""
    rng = np.random.default_rng(seed)
    sizes = 1 + rng.multinomial(n_obs - n_counties, np.full(n_counties, 1.0 / n_counties))
    county = np.repeat(np.arange(n_counties), sizes)
    rng.shuffle(county)
    floor = (rng.random(n_obs) < 0.17).astype(np.float64)
    a_c = rng.normal(1.5, 0.3, n_counties)
    b_c = rng.normal(-0.65, 0.3, n_counties)
    y = a_c[county] + b_c[county] * floor + rng.normal(0.0, 0.75, n_obs)
    return county.astype(np.int32), floor, y


def radon(n_obs: int = 919, n_counties: int = 85, seed: int = 123) -> ModelSpec:
    county, floor, y = radon_data(n_obs, n_counties, seed)
    J = n_counties
    vars_, n = _layout(
        [
            ("mu_a", "mu_a", 1, None, None),
            ("sigma_a_log__", "sigma_a", 1, "log", None),
            ("mu_b", "mu_b", 1, None, None),
            ("sigma_b_log__", "sigma_b", 1, "log", None),
            ("a", "a", J, None, None),
            ("b", "b", J, None, None),
            ("eps_log__", "eps", 1, "log", None),
        ]
    )
    ip = np.zeros(n)
    ip[1] = ip[3] = ip[n - 1] = np.log(5.0)
    return ModelSpec(
        KIND_RADON,
        n,
        vars_,
        data={"county_idx": county, "floor": floor, "y": y},
        meta={"n_counties": J, "n_obs": n_obs, "initial_point": ip},
    )


# ------------------------------------------------------------------------------------------------
# config 3: logistic GLM
# ------------------------------------------------------------------------------------------------
def logistic(n_rows: int = 1_000_000, n_features: int = 128, seed: int = 3) -> ModelSpec:
    """beta~Normal(0,1,K); y~Bernoulli(logit_p=X@beta)."""
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((n_rows, n_features))
    beta_true = rng.normal(0.0, 0.5, n_features)
    eta = X @ beta_true
    y = (rng.random(n_rows) < 1.0 / (1.0 + np.exp(-eta))).astype(np.uint8)
    vars_, n = _layout([("beta", "beta", n_features, None, None)])
    return ModelSpec(KIND_LOGISTIC, n, vars_, data={"X": X, "y": y}, meta={"n_rows": n_rows})


# ------------------------------------------------------------------------------------------------
# config 4: stochastic volatility, AR(1) latent log-variance
# ------------------------------------------------------------------------------------------------
def stochvol(T: int = 3000, seed: int = 4) -> ModelSpec:
    """mu~Normal(0,5); phi~Uniform(-1,1) [interval]; sigma~Exponential(10) [log];
    h~AR(rho=[phi], sigma, init_dist=Normal(0,1), shape=T); y~Normal(0, exp((mu+h)/2))."""
    rng = np.random.default_rng(seed)
    mu, phi, sigma = -1.0, 0.97, 0.15
    h = np.empty(T)
    h[0] = rng.normal(0.0, sigma / np.sqrt(1 - phi * phi))
    for t in range(1, T):
        h[t] = phi * h[t - 1] + sigma * rng.normal()
    y = rng.normal(0.0, 1.0, T) * np.exp(0.5 * (mu + h))
    vars_, n = _layout(
        [
            ("mu", "mu", 1, None, None),
            ("phi_interval__", "phi", 1, "interval", (-1.0, 1.0)),
            ("sigma_log__", "sigma", 1, "log", None),
            ("h", "h", T, None, None),
        ]
    )
    ip = np.zeros(n)
    ip[2] = np.log(0.1)  # Exponential(lam=10) support point is its mean 1/lam
    return ModelSpec(KIND_STOCHVOL, n, vars_, data={"y": y}, meta={"T": T, "initial_point": ip})


# ------------------------------------------------------------------------------------------------
# config 5: correlated Gaussian, dense covariance
# ------------------------------------------------------------------------------------------------
def mvgauss(n: int = 10_000, seed: int = 5, cache_dir: str | None = None) -> ModelSpec:
    """x~MvNormal(0, chol=L).  Stores L, Sigma=L L^T, the precision P=Sigma^-1 (the gradient is -P x) and L^-T (momentum
    draws of the dense mass matrix).  ``cache_dir``: keep the four n x n matrices on disk (e.g. /dev/shm) -- building them
    for n = 10^4 costs about a minute of BLAS time, and every rank of a multi-GPU run needs them."""
    import os

    import scipy.linalg as sl

    path = os.path.join(cache_dir, f"b200_mvgauss_n{n}_s{seed}.npz") if cache_dir else None
    if path and os.path.isfile(path):
        z = np.load(path)
        L, cov, P, LinvT, logdet = z["L"], z["cov"], z["prec"], z["LinvT"], float(z["logdet_L"])
    else:
        rng = np.random.default_rng(seed)
        d = np.exp(rng.normal(0.0, 0.5, n))
        L = np.tril(rng.standard_normal((n, n)), -1) * (0.05 / np.sqrt(n))
        L[np.diag_indices(n)] = d
        Linv = sl.solve_triangular(L, np.eye(n), lower=True)
        P = Linv.T @ Linv
        P = 0.5 * (P + P.T)
        cov = L @ L.T
        cov = 0.5 * (cov + cov.T)
        LinvT = np.ascontiguousarray(Linv.T)
        logdet = float(np.sum(np.log(d)))
        if path:
            try:
                os.makedirs(cache_dir, exist_ok=True)
                tmp = f"{path}.{os.getpid()}.tmp.npz"
                np.savez(tmp, L=L, cov=cov, prec=P, LinvT=LinvT, logdet_L=logdet)
                os.replace(tmp, path)
            except OSError:
                pass
    vars_, n_ = _layout([("x", "x", n, None, None)])
    return ModelSpec(
        KIND_MVGAUSS,
        n_,
        vars_,
        data={"L": L, "cov": cov, "prec": P, "LinvT": LinvT},
        meta={"logdet_L": logdet},
    )


BUILDERS = {
    "std_normal": std_normal,
    "eight_schools": eight_schools,
    "radon": radon,
    "logistic": logistic,
    "stochvol": stochvol,
    "mvgauss": mvgauss,
}
