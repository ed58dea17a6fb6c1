"""Shared helpers for the parity tests (tests may import oracle/; the product never does), and for the kernel tests that
call single entry points of the library against float64 (fp32/bf16/fp16 rounding, canary-guarded output buffers,
bounds and bitwise comparisons)."""
from types import SimpleNamespace

import numpy as np
import torch


def make_args(device, batch=32, cfg=None, rainbow_only=False, nb_actor=1, actor_capacity=1000):
    cfg = cfg or {}
    return SimpleNamespace(
        multi_step=cfg.get("n_step", 3), history_length=4, discount=cfg.get("discount", 0.99), device=device,
        batch_size=batch, length_actor_buffer=1000, model=None, lr=6.25e-5 if rainbow_only else 5e-5,
        adam_eps=1.5e-4 if rainbow_only else 3.125e-4, rainbow_only=int(rainbow_only), atoms=51, V_min=-10.0,
        V_max=10.0, kappa=cfg.get("kappa", 1.0), num_tau_samples=cfg.get("n_tau", 64),
        num_tau_prime_samples=cfg.get("n_tau_prime", 64), num_quantile_samples=cfg.get("n_quantile", 32),
        quantile_embedding_dim=64, hidden_size=512, noisy_std=0.1, disable_cuda=False, nb_actor=nb_actor,
        actor_capacity=actor_capacity, priority_weight=0.4, priority_exponent=0.2)


def load_params(net, params):
    """Load a numpy parameter blob (oracle.network.make_params) into a DQN through load_state_dict."""
    sd = {k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in params.items()}
    net.load_state_dict(sd)
    net.compose_weights()


def rel_err(a, b):
    a = np.asarray(a, np.float64)
    b = np.asarray(b, np.float64)
    return float(np.max(np.abs(a - b)) / (np.max(np.abs(b)) + 1e-30))


def digest(t, head=8):
    a = t.detach().cpu().numpy().astype(np.float64).ravel()
    return np.concatenate([[a.sum(), np.abs(a).sum(), np.sqrt((a * a).sum())], a[:head]])


# ---------------------------------------------------------------------------------------------- kernel-test helpers
U = 2.0 ** -24          # unit roundoff of fp32
PAD = 512               # canary elements past the end of every output buffer
CANARY = -77.0          # exact in fp32, bf16 and fp16


def bf16_bits(x):
    """float32 -> bf16 bit patterns, round to nearest even (finite inputs)."""
    u = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32)
    return ((u + (((u >> 16) & 1) + np.uint32(0x7FFF))) >> 16).astype(np.uint16)


def bf16(x):
    """float32 values rounded to bf16 (returned as float32)."""
    return (bf16_bits(x).astype(np.uint32) << 16).view(np.float32)


def f16_bits(x):
    """float32 -> fp16 bit patterns, round to nearest even (overflow -> inf, as the device conversion)."""
    with np.errstate(over="ignore"):
        return np.ascontiguousarray(x, dtype=np.float32).astype(np.float16).view(np.uint16)


def f32_bits(x):
    return np.ascontiguousarray(x, dtype=np.float32).view(np.uint32)


def lib_call(name, *args):
    from rainbow_iqn_apex_b200._lib import call
    call(name, *args)


def dptr(t):
    return None if t is None else t.data_ptr()


def to_dev(a, dev, dtype=torch.float32):
    return torch.from_numpy(np.ascontiguousarray(a)).to(device=dev, dtype=dtype)


def to_dev_bf16(x, dev):
    """Device bf16 tensor holding bf16(x) (x float32)."""
    return torch.from_numpy(bf16_bits(x).view(np.int16)).to(dev).view(torch.bfloat16)


class Out:
    """A flat output buffer of n elements followed by PAD canaries."""

    def __init__(self, n, dev, dtype=torch.float32, fill=float("nan")):
        self.n = n
        self.t = torch.full((n + PAD,), CANARY, dtype=dtype, device=dev)
        if isinstance(fill, np.ndarray):
            self.t[:n] = torch.from_numpy(np.ascontiguousarray(fill, np.float32).ravel()).to(dev, dtype)
        else:
            self.t[:n].fill_(fill)

    @property
    def p(self):
        return self.t.data_ptr()

    def canaries_ok(self):
        return bool(torch.all(self.t[self.n:] == CANARY))

    def f32(self):
        return self.t[:self.n].float().cpu().numpy()

    def bits(self):
        """bit patterns of the body: uint16 for 16-bit buffers, uint32 for fp32"""
        body = self.t[:self.n]
        if body.element_size() == 2:
            return body.view(torch.int16).cpu().numpy().view(np.uint16)
        return body.view(torch.int32).cpu().numpy().view(np.uint32)


def assert_canaries(outs):
    bad = [k for k, o in outs.items() if o is not None and not o.canaries_ok()]
    assert not bad, f"writes past the end of {bad}"


def check_bound(what, got, ref, bound):
    """|got - ref| <= bound elementwise; prints and returns the worst err/bound ratio."""
    got = np.asarray(got, np.float64)
    ref = np.asarray(ref, np.float64)
    assert np.all(np.isfinite(got)), f"{what}: non-finite values"
    err = np.abs(got - ref)
    bound = np.asarray(bound, np.float64) + 1e-300
    ratio = err / bound
    worst = float(ratio.max()) if ratio.size else 0.0
    print(f"{what}: worst err/bound {worst:.3g}")
    if worst > 1.0:
        i = np.unravel_index(int(np.argmax(ratio)), ratio.shape)
        raise AssertionError(f"{what}: at {i} got {got[i]!r} ref {ref[i]!r} bound {bound[i]!r}")
    return worst


def assert_bits(what, got, want):
    got, want = np.asarray(got), np.asarray(want)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    bad = got != want
    if bad.any():
        i = np.argwhere(bad)[0]
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.size} elements differ, first at {tuple(i)}: "
                             f"got {got[tuple(i)]:#x} want {want[tuple(i)]:#x}")


def prefill_pattern(n, scale=0.25, mod=13):
    """A non-zero prefill for accumulated outputs, exact in fp32."""
    return (((np.arange(n) % mod) - mod // 2) * scale + scale / 2).astype(np.float32)


_M32 = np.uint64(0xFFFFFFFF)


def philox_np(seed, stream, count):
    """Philox4x32-10 (Salmon et al. 2011) words of counters 0 .. count-1 under (seed, stream), in the order
    riqn_fill_uniform consumes them: word 4i + j is component j of draw i.  (count * 4,) uint32."""
    idx = np.arange(count, dtype=np.uint64)
    c = [idx & _M32, idx >> np.uint64(32), np.full(count, stream & 0xFFFFFFFF, np.uint64),
         np.full(count, stream >> 32, np.uint64)]
    k0, k1 = np.uint64(seed & 0xFFFFFFFF), np.uint64(seed >> 32)
    for _ in range(10):
        p0, p1 = np.uint64(0xD2511F53) * c[0], np.uint64(0xCD9E8D57) * c[2]
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ k0, p1 & _M32, (p0 >> np.uint64(32)) ^ c[3] ^ k1, p0 & _M32]
        k0, k1 = (k0 + np.uint64(0x9E3779B9)) & _M32, (k1 + np.uint64(0xBB67AE85)) & _M32
    return np.stack(c, 1).astype(np.uint32).ravel()
