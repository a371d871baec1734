"""Reference of tempered ladders (DESIGN.md §2 "Tempered ladders"), restated over the oracle's primitives: the same Philox stream
(orc_stream_uniform, orc_rnorm, orc_shuffle), the same Math.exp / Math.log (orc_exp, orc_log), and the steppers of
oracle/amwg_oracle.c (onedim_step, binary_step, multidim_step, amwg_step) with one change each, the rung's beta:

    onedim:  accept_prob = Math.exp(beta * (prop_log_dens - curr_log_dens))
    binary:  zero_log_dens, one_log_dens = beta * log_post(state with 0), beta * log_post(state with 1), then as the reference

With beta = 1 a RefChain is the oracle's chain (tests/test_temper_host.py holds it to orc_create/orc_step chain for chain). A RefLadder
steps every chain once, then runs swap round k exactly as the device: in every ladder each rung r = k (mod 2), r + 1 < K exchanges its
state with rung r + 1 iff Math.exp((beta_r - beta_{r+1}) * (lp_{r+1} - lp_r)) > uniform #(2^63 + 2^62 + k) of rung r's stream.
TEST INFRASTRUCTURE ONLY: nothing under bayes.js_b200/ imports it."""
from __future__ import annotations

import ctypes as C
import math
from typing import Callable, Dict, List, Optional

import numpy as np

SWAP_STREAM_BASE = (1 << 63) + (1 << 62)


def js_max(a: float, b: float) -> float:
    if a != a or b != b:
        return math.nan
    return a if a > b else b


def js_min(a: float, b: float) -> float:
    if a != a or b != b:
        return math.nan
    return a if a < b else b


def swap_accept(O, beta_a: float, beta_b: float, lp_a: float, lp_b: float, u: float) -> bool:
    return O.orc_exp((beta_a - beta_b) * (lp_b - lp_a)) > u


def swap_uniform(O, seed: int, chain_a: int, rnd: int) -> float:
    return O.orc_stream_uniform(seed, chain_a, SWAP_STREAM_BASE + rnd)


class RefChain:
    """One chain of the reference sampler at inverse temperature `beta`. f(x) -> log_post, where x has D + n_derived slots and f may
    write the derived ones (as an oracle closure)."""

    def __init__(self, orc, f: Callable, params: Dict[str, dict], seed: int, chain: int, beta: float = 1.0, n_derived: int = 0,
                 comp_options: Optional[Dict[str, dict]] = None):
        self.O = orc.lib()
        cp, prm, init, opts, D = orc._layout(params, comp_options)
        self.f, self.seed, self.chain, self.beta, self.D = f, int(seed), int(chain), float(beta), D
        self.x = np.zeros(D + n_derived)
        self.x[:D] = init
        self.n_derived = n_derived
        self.n = C.c_uint64(0)
        self.params = [(prm[p].type, prm[p].n_comp, prm[p].dim0, prm[p].comp_offset, prm[p].lower, prm[p].upper) for p in range(len(prm))]
        self.order = list(range(len(self.params)))
        self.pls = np.array([opts[c].prop_log_scale for c in range(D)])
        self.batch_size = np.array([opts[c].batch_size for c in range(D)])
        self.max_adapt = np.array([opts[c].max_adaptation for c in range(D)])
        self.init_adapt = np.array([opts[c].initial_adaptation for c in range(D)])
        self.target = np.array([opts[c].target_accept_rate for c in range(D)])
        self.adapting = np.array([bool(opts[c].is_adapting) for c in range(D)])
        self.acc = np.zeros(D)
        self.iters = np.zeros(D)
        self.batches = np.zeros(D)
        for p in self.params:                       # binary components have no OnedimMetropolisStepper
            if p[0] == 2:
                self.adapting[p[3]:p[3] + p[1]] = False
        self.f(self.x)

    def log_post(self) -> float:
        return float(self.f(self.x))

    def _u(self) -> float:
        u = self.O.orc_stream_uniform(self.seed, self.chain, self.n.value)
        self.n.value += 1
        return u

    def _onedim(self, c: int, is_int: bool, lower: float, upper: float):
        O = self.O
        cur = self.x[c]
        prop = O.orc_rnorm(self.seed, self.chain, C.byref(self.n), cur, O.orc_exp(self.pls[c]))
        if is_int:
            prop = O.orc_js_round(prop)
        if not (prop < lower or prop > upper):
            curr_ld = self.log_post()
            self.x[c] = prop
            prop_ld = self.log_post()
            accept_prob = O.orc_exp(self.beta * (prop_ld - curr_ld))
            if accept_prob > self._u():
                if self.adapting[c]:
                    self.acc[c] += 1
            else:
                self.x[c] = cur
        if self.adapting[c]:
            self.iters[c] += 1
            if self.iters[c] >= self.batch_size[c]:
                self.batches[c] += 1
                adj = js_min(self.max_adapt[c], self.init_adapt[c] / math.sqrt(self.batches[c]))
                if self.acc[c] / self.batch_size[c] > self.target[c]:
                    self.pls[c] += adj
                else:
                    self.pls[c] -= adj
                self.acc[c] = 0
                self.iters[c] = 0

    def _binary(self, c: int):
        O = self.O
        self.x[c] = 0
        z0 = self.beta * self.log_post()
        self.x[c] = 1
        z1 = self.beta * self.log_post()
        mx = js_max(z0, z1)
        z0, z1 = z0 - mx, z1 - mx
        zero_prob = O.orc_exp(z0 - O.orc_log(O.orc_exp(z0) + O.orc_exp(z1)))
        if self._u() < zero_prob:
            self.x[c] = 0

    def step(self):
        P = len(self.params)
        for i in range(P - 1, 0, -1):               # shuffle_array(this.substeppers), in place
            j = int(math.floor(self._u() * (i + 1)))
            self.order[i], self.order[j] = self.order[j], self.order[i]
        for p in self.order:
            ptype, n_comp, dim0, off, lower, upper = self.params[p]
            if n_comp == 1 and dim0 == 1:
                if ptype == 2:
                    self._binary(off)
                else:
                    self._onedim(off, ptype == 1, lower, upper)
                continue
            inner = n_comp // dim0
            idx = (C.c_int * dim0)(*range(dim0))
            self.O.orc_shuffle(self.seed, self.chain, C.byref(self.n), C.cast(idx, C.c_void_p), dim0)
            for i in range(dim0):
                for r in range(inner):
                    c = off + idx[i] * inner + r
                    if ptype == 2:
                        self._binary(c)
                    else:
                        self._onedim(c, ptype == 1, lower, upper)
        if self.n_derived > 0:
            self.f(self.x)


class RefLadder:
    """ladders x K RefChains: global chains first_chain .. first_chain + ladders K - 1, chain g at beta[g mod K]."""

    def __init__(self, orc, f: Callable, params: Dict[str, dict], seed: int, betas: List[float], ladders: int, first_chain: int = 0,
                 n_derived: int = 0, comp_options: Optional[Dict[str, dict]] = None):
        self.O = orc.lib()
        self.K, self.betas, self.seed, self.first_chain = len(betas), [float(b) for b in betas], int(seed), int(first_chain)
        assert first_chain % self.K == 0
        self.chains = [RefChain(orc, f, params, seed, first_chain + g, self.betas[(first_chain + g) % self.K], n_derived, comp_options)
                       for g in range(ladders * self.K)]
        self.rounds = 0
        self.accepts = np.zeros((ladders, self.K - 1), dtype=np.int64)

    def swap_round(self):
        K, k = self.K, self.rounds
        for ell in range(len(self.chains) // K):
            for r in range(k & 1, K - 1, 2):
                a, b = self.chains[ell * K + r], self.chains[ell * K + r + 1]
                u = swap_uniform(self.O, self.seed, a.chain, k)
                if swap_accept(self.O, self.betas[r], self.betas[r + 1], a.log_post(), b.log_post(), u):
                    a.x, b.x = b.x, a.x                 # the state (and its derived slots) changes hands; the rest stays
                    self.accepts[ell, r] += 1
        self.rounds += 1

    def step(self):
        for ch in self.chains:
            ch.step()
        self.swap_round()

    def burn(self, n: int):
        for _ in range(n):
            self.step()

    def sample(self, n: int, entries: List[int], thin: int = 1) -> np.ndarray:
        """[rows, len(entries), ladders]: the rung-0 chains, recorded before each kept sweep"""
        cold = self.chains[::self.K]
        rows = []
        for i in range(n):
            if i % thin == 0:
                rows.append(np.stack([ch.x[entries] for ch in cold], axis=1))
            self.step()
        return np.asarray(rows)

    def states(self) -> np.ndarray:
        return np.stack([ch.x for ch in self.chains])
