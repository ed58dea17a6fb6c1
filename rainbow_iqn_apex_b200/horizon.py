"""Update-horizon and discount annealing (BBF, Schwarzer et al., "Bigger, Better, Faster: Human-level Atari with
human-level efficiency", ICML 2023): under ``horizon_anneal`` the learner's n-step horizon n and discount gamma start at
(horizon_anneal_n, horizon_anneal_gamma) after every reset (or construction) and reach (multi_step, discount) after
horizon_anneal_steps updates.  BBF's values are n from 10 down to 3 and gamma from 0.97 up to 0.997 over 10k steps.

The schedule is this project's reading of BBF's "exponential annealing", log-linear in n and in 1 - gamma; it is not
taken from BBF's code.  With u the updates since the last reset, P = horizon_anneal_steps and f = clamp((P - u) / P, 0,
1), in float64:

    n_u     = floor(exp(f ln n0 + (1 - f) ln n1) + 0.5)
    gamma_u = 1 - exp(f ln(1 - gamma0) + (1 - f) ln(1 - gamma1))

and at f = 1 and f = 0 the end values themselves, so that the end of the schedule is exactly the fixed configuration.

A step reads (n_u, gamma_u) on the device (dynstate.HorizonState): the sampler's valid-index shift and the transition
assembly at n_u (ReplayMemory.sample_horizon), which also forms each transition's discount fl32(gamma_u^n_u) * nt.  The
loss kernels take those discounts in place of the nonterminals with gamma^n = 1 (Agent.gamma_n), and compute the same
bootstrap factor bit for bit, so none of them changed.
"""
import math


def schedule(anneal, n1, gamma1, u):
    """(n_u, gamma_u) of the schedule ``anneal`` = (n0, gamma0, P) towards (n1, gamma1) after ``u`` updates."""
    n0, gamma0, steps = anneal
    f = min(max((steps - u) / steps, 0.0), 1.0)
    if f == 0.0:
        return n1, gamma1
    if f == 1.0:
        return n0, gamma0
    n = math.floor(math.exp(f * math.log(n0) + (1.0 - f) * math.log(n1)) + 0.5)
    gamma = 1.0 - math.exp(f * math.log(1.0 - gamma0) + (1.0 - f) * math.log(1.0 - gamma1))
    return int(n), gamma
