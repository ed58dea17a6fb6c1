"""Oracle (test infrastructure): the distortion risk measures of risk-sensitive IQN policies, in float64.

Dabney, Ostrovski, Silver, Munos, "Implicit Quantile Networks for Distributional Reinforcement Learning", ICML 2018,
section 3.1: an agent acts greedily on Q_beta(x, a) = mean_k Z_{beta(tau_k)}(x, a), tau_k ~ U(0, 1), with

  CVaR(eta)  beta(t) = eta t                                             (0 < eta <= 1)
  Wang(eta)  beta(t) = Phi(Phi^-1(t) + eta)                              (eta < 0 risk-averse, eta > 0 risk-seeking)
  CPW(eta)   beta(t) = t^eta / (t^eta + (1 - t)^eta)^(1/eta)             (eta > 0; Tversky & Kahneman's weighting)
  Pow(eta)   beta(t) = t^(1/(1+|eta|)) if eta >= 0 else 1 - (1 - t)^(1/(1+|eta|))
  Norm(eta)  the mean of eta independent uniforms                        (eta = 1, 2, ...)

The reference implements none of them, so there is no golden fixture: tests check this module by the identities of the
functions (identity parameters, monotonicity, the risk-averse / risk-seeking orderings).
"""
import numpy as np
from scipy.special import ndtr, ndtri


def distort(measure, eta, u):
    """beta(u) in float64.  ``u``: uniforms in (0, 1).  For "norm", ``u`` holds eta uniforms per output: shape (n, eta),
    or a flat array of n * eta values taken eta at a time in order; they are summed left to right, then divided by eta."""
    u = np.asarray(u, np.float64)
    eta = float(eta)
    if measure == "neutral":
        return u.copy()
    if measure == "cvar":
        return eta * u
    if measure == "wang":
        return ndtr(ndtri(u) + eta)
    if measure == "cpw":
        a = np.power(u, eta)
        return a / np.power(a + np.power(1.0 - u, eta), 1.0 / eta)
    if measure == "pow":
        e = 1.0 / (1.0 + abs(eta))
        return np.power(u, e) if eta >= 0 else 1.0 - np.power(1.0 - u, e)
    if measure == "norm":
        m = int(eta)
        g = u.reshape(-1, m)
        s = np.zeros(g.shape[0])
        for j in range(m):                       # left to right, like the device's loop
            s = s + g[:, j]
        return s / eta
    raise ValueError(measure)
