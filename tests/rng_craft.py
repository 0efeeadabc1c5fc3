"""Crafted numpy PCG64 states: generator states whose output number m is a chosen 64-bit word.

numpy's PCG64 steps its 128-bit state s -> A s + inc (mod 2^128) and then outputs the XSL-RR permutation of the NEW
state, rotr(hi ^ lo, hi >> 58).  For a chosen word X and a chosen high half `hi`, lo = rotl(X, hi >> 58) ^ hi gives
a state that outputs X; stepping it back m + 1 times with A^-1 gives the state whose output m is X, for any odd
increment.  That reaches the draws a random seed hits with probability 2^-32 or less: a 32-bit word 0 (rejected by
Lemire's bounded integers for every n that is not a power of two) and the ziggurat's wedge and tail.

The words are exchanged in the HwyHighwayState.rng layout: [state_hi, state_lo, inc_hi, inc_lo,
has_uint32 << 32 | uinteger].
"""
from __future__ import annotations

import numpy as np

M64 = (1 << 64) - 1
M128 = (1 << 128) - 1
PCG_MULT = (0x2360ED051FC65DA4 << 64) | 0x4385DF649FCCF645
PCG_MULT_INV = pow(PCG_MULT, -1, 1 << 128)
ZIGGURAT_NOR_R = 3.6541528853610088  # numpy ziggurat_nor_r: |x| >= R only through the tail


def rotl64(x: int, r: int) -> int:
    r &= 63
    return ((x << r) | (x >> (64 - r))) & M64 if r else x


def output_of(state: int) -> int:
    """XSL-RR output of a (post-step) 128-bit state."""
    hi, lo = state >> 64, state & M64
    r = hi >> 58
    x = hi ^ lo
    return ((x >> r) | (x << (64 - r))) & M64 if r else x


def state_emitting(x: int, hi: int) -> int:
    """The post-step state with high half `hi` whose output is x."""
    return (hi << 64) | (rotl64(x, hi >> 58) ^ hi)


def step_back(state: int, inc: int, m: int = 1) -> int:
    for _ in range(m):
        state = ((state - inc) * PCG_MULT_INV) & M128
    return state


def crafted_state(x: int, inc: int, m: int = 0, hi: int | None = None, seed: int = 0) -> int:
    """A 128-bit state whose output number m (0 = the next next64()) is x, under increment inc (odd)."""
    assert inc & 1, "PCG64 increments are odd"
    if hi is None:
        hi = int(np.random.default_rng(seed).integers(0, 1 << 63, dtype=np.uint64)) << 1 | 1
    return step_back(state_emitting(x, hi), inc, m + 1)


def make_generator(state: int, inc: int, has_uint32: int = 0, uinteger: int = 0) -> np.random.Generator:
    bg = np.random.PCG64()
    bg.state = {"bit_generator": "PCG64", "state": {"state": int(state), "inc": int(inc)},
                "has_uint32": int(has_uint32), "uinteger": int(uinteger)}
    return np.random.Generator(bg)


def seeded_state(seed: int) -> tuple[int, int]:
    """(state, inc) of Generator(PCG64(SeedSequence(seed))), the env seeding."""
    st = np.random.PCG64(np.random.SeedSequence(int(seed))).state["state"]
    return int(st["state"]), int(st["inc"])


def words_of(gen_or_state, inc: int | None = None, has_uint32: int = 0, uinteger: int = 0) -> np.ndarray:
    """The 5 rng words [uint64] of a Generator / PCG64 or of (state, inc, has_uint32, uinteger)."""
    if inc is None:
        bg = getattr(gen_or_state, "bit_generator", gen_or_state)
        st = bg.state
        state, inc = st["state"]["state"], st["state"]["inc"]
        has_uint32, uinteger = st["has_uint32"], st["uinteger"]
    else:
        state = gen_or_state
    return np.array([state >> 64, state & M64, inc >> 64, inc & M64, (int(has_uint32) << 32) | int(uinteger)],
                    dtype=np.uint64)


def generator_of(words) -> np.random.Generator:
    w = [int(v) for v in np.asarray(words, dtype=np.uint64)]
    return make_generator((w[0] << 64) | w[1], (w[2] << 64) | w[3], w[4] >> 32, w[4] & 0xFFFFFFFF)


# ---- 64-bit words that steer the ziggurat of Generator.standard_normal (random_standard_normal, distributions.c):
# bits 0-7 the layer, bit 8 the sign, bits 9-60 the magnitude; a magnitude >= ki[layer] leaves the fast path.  The
# largest magnitude is >= ki[layer] for every layer: layer 0 then samples the tail, any other layer the wedge.
def ziggurat_word(layer: int, negative: bool = False, magnitude: int = (1 << 52) - 1) -> int:
    return (magnitude << 9) | (int(negative) << 8) | (layer & 0xFF)


def ziggurat_tail_word(negative: bool) -> int:
    """Layer 0 at a large magnitude: the tail, whose sign is bit 8 of the magnitude (not the sign bit)."""
    return ziggurat_word(0, magnitude=((1 << 52) - 1) & ~(1 << 8) | (int(negative) << 8))


def lemire_rejects(r32: int, n: int) -> bool:
    """Does Lemire's method (numpy random_buffered_bounded_lemire_uint32, rng = n - 1) reject the 32-bit word r32?"""
    m = r32 * n
    leftover = m & 0xFFFFFFFF
    return leftover < n and leftover < ((1 << 32) - n) % n


def spawn_requests(n_vehicles: int, lanes_count: int, has_uint32: int, ego_draws_lane: bool = True):
    """Where HighwayEnv._create_vehicles' lane choices come from, in draw order, assuming no rejection: a list of
    (vehicle, output index, 'low' | 'high' | 'buffered').  Vehicle.create_random draws choice(lanes) (one 32-bit
    request when lanes > 1) then its 64-bit uniforms: 1 for the ego (position) and 3 for traffic (speed, position,
    DELTA)."""
    out, nxt, has, opened = [], 0, bool(has_uint32), -1
    for v in range(n_vehicles):
        if lanes_count > 1 and (v > 0 or ego_draws_lane):
            if has:
                out.append((v, opened, "high") if opened >= 0 else (v, -1, "buffered"))
                has = False
            else:
                out.append((v, nxt, "low"))
                opened, nxt, has = nxt, nxt + 1, True
        nxt += 1 if v == 0 else 3
    return out
