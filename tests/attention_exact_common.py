"""Exact-weight inputs of the softmax attention (softmax_attention.cuh) and their fp64 reference.

The kernel rounds the softmax weights P = 2^(s - m + 14) to fp16 (softmax_tile), an unbiased ~1e-4 perturbation of a
general softmax, so random inputs only allow bars near 1e-4.  These inputs make that rounding exact:
  * a query of group g is alpha e_g, a member key of group g at level n is beta_n e_g, every other key is zero;
  * the score the kernel forms, fp32(alpha * fp32(scale * log2 e)) * beta_n, is within LEVEL_TOL of L - n (L in 55..60),
    so fp16(2^(s - m + 14)) is exactly 2^(14 - n): the fp16 spacing allows 3.5e-4 below a power of two;
  * non-members score 0, at least GAP below the level-0 score: 2^(14 - GAP) rounds to 0 in fp16.  A query whose group
    has no member sees all N keys at score exactly 0, weight 1.
On them the kernel computes sum(w v) / sum(w) with known power-of-two weights, and what is left is V's hi + lo split,
the tensor core's fp32 sums and the fold: an fp32-class error.

The online softmax rescales what it has summed when a later key tile raises a row's maximum, by ex2(m_old - m), which
is not exact.  So in every key range a CTA covers (all keys, or a part of the split plan) a group's first tile with
members holds a level-0 member of the group (its anchor), or the range holds no member of it at all; such a part's
partial has m = 0 and is merged with weight 2^-L.

Three patterns are mixed in every input, by group: uniform (no members), ties (several bitwise-equal level-0 members
scattered over the key tiles) and levels (members at levels 0..8, weights 2^-n).  Members sit at key 0, key N - 1 (the
only member of a partial last tile), the first and last tile of every key range and random keys.  In the ViT layout
every image has the same queries and keys and its own values, so another image's members are decoys that only the
image row map keeps out."""
import ctypes
from dataclasses import dataclass, field

import numpy as np

LOG2E = 1.4426950408889634   # csrc: scale * 1.4426950408889634f, the kernel works in log2 units
P_BIAS = 14.0                # softmax_tile: P = fp16(2^(s - m + 14))
MASK = -1e30                 # softmax_tile: score of a key >= N
VIT_SCALE = 0.125            # vit.cu: head_dim ** -0.5
STAGE1_SCALE = 0.25          # a fixed scale (log(N, 12185) is 0 at N = 1)
LEVEL_TOL = 5e-5             # |score - (L - n)| of a member, log2 units
GAP = 44                     # non-members score at least this much below level 0
SCORE_MAX = 64.0
LEVELS = 9                   # levels 0..8: weights 1 .. 2^-8
TILE = 128                   # keys per tile


@dataclass(frozen=True)
class Geometry:
    heads: int
    hd: int
    q: int     # first column of Q, K and V in a qkv row
    k: int
    v: int


STAGE1 = Geometry(4, 16, 0, 64, 128)      # qkv [N][3][4][16]
VIT = Geometry(12, 64, 0, 768, 1536)      # qkv [n N][ldq >= 2304] = [q | k | v] x 12 heads x 64


def qscale(scale):
    """the factor qkv_tile_kernel / vit_qkv_tile_kernel multiply Q by, in fp32"""
    return np.float32(np.float32(scale) * np.float32(LOG2E))


def combos(scale):
    """(alpha, beta_0, L) with alpha and beta_0 fp16-exact and fp32(alpha * qscale) * beta_0 within LEVEL_TOL of L,
    best first"""
    qs = qscale(scale)
    alphas = np.arange(np.float16(2.0).view(np.uint16), np.float16(16.0).view(np.uint16), dtype=np.uint16).view(np.float16)
    qp = (alphas.astype(np.float32) * qs).astype(np.float64)
    out = []
    for L in range(55, 61):
        b0 = (L / qp).astype(np.float16).astype(np.float64)
        err = np.abs(qp * b0 - L)
        for i in np.nonzero(err < LEVEL_TOL / 4)[0]:
            out.append((float(err[i]), float(alphas[i]), float(b0[i]), L))
    out.sort()
    assert len(out) >= 4, "no exact (alpha, beta_0, L)"
    return [c[1:] for c in out]


def betas(alpha, L, scale):
    """beta_n, n = 0..8, fp32: beta_0 is the fp16-exact one of combos()"""
    qp = float(np.float32(np.float32(alpha) * qscale(scale)))
    return np.array([np.float16(L / qp) if n == 0 else np.float32((L - n) / qp) for n in range(LEVELS)], np.float32)


def split_plan(N, sms):
    """(split items, parts) of mvsf_attention_split_plan for N tokens on sms SMs (a host function)"""
    from mvsformerplusplus_b200 import _lib
    r, k = ctypes.c_int(), ctypes.c_int()
    _lib.call("mvsf_attention_split_plan", N, sms, ctypes.byref(r), ctypes.byref(k))
    return r.value, k.value


def key_ranges(N, plan):
    """the key-tile ranges [t0, t1) of the parts of a split item (attention_fa_kernel); [(0, ntiles)] without a split"""
    ntiles = -(-N // TILE)
    r, k = plan
    if not r:
        return [(0, ntiles)]
    return [(p * ntiles // k, (p + 1) * ntiles // k) for p in range(k)]


@dataclass
class Case:
    geo: Geometry
    n: int              # images (1 for stage-1)
    N: int              # tokens per image
    scale: float
    qkv: np.ndarray     # fp32 [n N][ldq]
    qgroup: np.ndarray  # [heads][N] group of query t
    kgroup: np.ndarray  # [heads][N] group of key t, -1: not a member
    klevel: np.ndarray  # [heads][N]
    L: list             # per head
    ranges: list        # key-tile ranges of the split plan's parts (all keys: [(0, ntiles)])
    kinds: dict = field(default_factory=dict)   # (head, group) -> "uniform" | "ties" | "levels"

    def cols(self, which, h):
        c = {"q": self.geo.q, "k": self.geo.k, "v": self.geo.v}[which] + h * self.geo.hd
        return slice(c, c + self.geo.hd)

    def members(self, h, g):
        return np.nonzero(self.kgroup[h] == g)[0]


def _head(geo, N, h, ranges, rng):
    """query groups, key groups and levels of head h"""
    G = geo.hd
    kind = {g: ("uniform", "ties", "levels")[(g + h) % 3] for g in range(G)}
    kg = np.full(N, -1, np.int64)
    kl = np.zeros(N, np.int64)
    ntiles = -(-N // TILE)
    # a partial last tile that starts no range holds one member only, at key N - 1
    last_start = TILE * (ntiles - 1)
    lonely = N % TILE != 0 and all(t0 != ntiles - 1 for t0, _ in ranges)

    def put(t, g, n):
        if 0 <= t < N and kg[t] < 0:
            kg[t], kl[t] = g, n
            return True
        return False

    member_groups = [g for g in range(G) if kind[g] != "uniform"]
    present = {}   # range index -> groups with members in it
    for p, (t0, t1) in enumerate(ranges):
        lo, hi = TILE * t0, min(TILE * t1, N)
        present[p] = []
        for i, g in enumerate(member_groups):
            if p > 0 and (g not in present[0] or (g + p) % 2):
                continue          # no member of g in this part: its partial is merged with weight 2^-L
            if lo + i < hi and put(lo + i, g, 0):       # the anchor, in the range's first tile
                present[p].append(g)
    for g in member_groups:
        if g not in present[0]:
            kind[g] = "uniform"   # no room for its anchor in tile 0 (N small)
    for p, (t0, t1) in enumerate(ranges):
        lo, hi = TILE * t0, min(TILE * t1, N)
        top = min(hi, last_start) if lonely else hi     # random members stay out of a lonely last tile
        tail_lo = max(lo, TILE * (t1 - 1))
        for g in present[p]:
            levels = [0, 0, 0] if kind[g] == "ties" else list(range(1, LEVELS))
            for n in levels:
                for _ in range(8 if top > lo else 0):   # a few draws past keys already taken
                    if put(int(rng.integers(lo, top)), g, n):
                        break
            if tail_lo < min(hi, top):                   # the range's last tile
                put(int(rng.integers(tail_lo, min(hi, top))), g, 0 if kind[g] == "ties" else int(rng.integers(1, LEVELS)))
    if kg[N - 1] < 0 and present[len(ranges) - 1]:
        g = present[len(ranges) - 1][0]
        put(N - 1, g, 0 if kind[g] == "ties" else 3)
    qg = (7 * np.arange(N) + 3 * h) % G
    return qg, kg, kl, kind


def make_case(geo, N, n=1, scale=None, plan=(0, 1), ldq=None, seed=0):
    """qkv and its intended weights.  plan: (split items, parts) of the split plan the kernel will run (stage-1)."""
    scale = STAGE1_SCALE if scale is None else scale
    ldq = ldq or (geo.v + geo.heads * geo.hd)
    rng = np.random.default_rng(seed)
    ranges = key_ranges(N, plan)
    cmb = combos(scale)
    qkv = np.full((n * N, ldq), np.nan, np.float32)     # columns past 3 x 768 (stage-1: none) are never read
    qkv[:, :geo.v + geo.heads * geo.hd] = 0.0
    H = geo.heads
    qgroup, kgroup, klevel, L, kinds = (np.zeros((H, N), np.int64), np.zeros((H, N), np.int64),
                                        np.zeros((H, N), np.int64), [], {})
    for h in range(H):
        alpha, _, Lh = cmb[h % len(cmb)]
        beta = betas(alpha, Lh, scale)
        qg, kg, kl, kind = _head(geo, N, h, ranges, rng)
        qgroup[h], kgroup[h], klevel[h] = qg, kg, kl
        L.append(Lh)
        kinds.update({(h, g): kind[g] for g in range(geo.hd)})
        for b in range(n):
            rows = slice(b * N, (b + 1) * N)
            q = np.zeros((N, geo.hd), np.float32)
            q[np.arange(N), qg] = alpha
            k = np.zeros((N, geo.hd), np.float32)
            m = kg >= 0
            k[np.nonzero(m)[0], kg[m]] = beta[kl[m]]
            qkv[rows, geo.q + h * geo.hd:geo.q + (h + 1) * geo.hd] = q
            qkv[rows, geo.k + h * geo.hd:geo.k + (h + 1) * geo.hd] = k
    v = rng.standard_normal((n * N, geo.heads * geo.hd)).astype(np.float32)   # every image its own values
    qkv[:, geo.v:geo.v + geo.heads * geo.hd] = v
    return Case(geo, n, N, scale, qkv, qgroup, kgroup, klevel, L, ranges, kinds)


def scores(case, h):
    """every distinct score of head h as the kernel forms it, fp64 from the fp32 inputs: (S [distinct queries][distinct
    keys], query index of each row, key index of each row)"""
    q = case.qkv[:, case.cols("q", h)] * qscale(case.scale)          # fp32 product, as the tiling kernels do
    k = case.qkv[:, case.cols("k", h)]
    uq, qi = np.unique(q.astype(np.float64), axis=0, return_inverse=True)
    uk, ki = np.unique(k.astype(np.float64), axis=0, return_inverse=True)
    return uq @ uk.T, qi.reshape(-1), ki.reshape(-1)


def intended_weights(case, h):
    """(S, w): the distinct scores of head h and the weight each is meant to get, w[u, j] = 2^-n for a member of the
    query's group, 1 for every key of a query whose group has none, 0 otherwise"""
    S, qi, ki = scores(case, h)
    N = case.N
    rows_g = np.tile(case.qgroup[h], case.n)
    keys_g, keys_l = np.tile(case.kgroup[h], case.n), np.tile(case.klevel[h], case.n)
    ug = np.full(S.shape[0], -1)
    ug[qi] = rows_g
    assert all(len(set(rows_g[qi == u])) == 1 for u in range(S.shape[0])), "a distinct query spans groups"
    ukg, ukl = np.full(S.shape[1], -2), np.zeros(S.shape[1], np.int64)
    ukg[ki], ukl[ki] = keys_g, keys_l
    for j in range(S.shape[1]):
        assert len(set(zip(keys_g[ki == j], keys_l[ki == j]))) == 1, "a distinct key spans groups or levels"
    has = {g: bool((case.kgroup[h] == g).any()) for g in range(case.geo.hd)}
    w = np.zeros_like(S)
    for u in range(S.shape[0]):
        g = ug[u]
        if has[g]:
            mem = ukg == g
            w[u, mem] = 2.0 ** -ukl[mem]
        else:
            w[u, :] = 1.0
    assert N > 0
    return S, w, ug, ukg, ukl, has


def premise(case):
    """asserts the inputs give the intended weights; returns the largest |member score - (L - n)|"""
    worst = 0.0
    for h in range(case.geo.heads):
        S, w, ug, ukg, ukl, has = intended_weights(case, h)
        L = case.L[h]
        assert np.abs(S).max() <= SCORE_MAX
        for u in range(S.shape[0]):
            g = ug[u]
            if not has[g]:
                assert (S[u] == 0).all(), (h, g, "a uniform row has a nonzero score")
                continue
            mem = ukg == g
            dev = np.abs(S[u, mem] - (L - ukl[mem]))
            assert dev.max() <= LEVEL_TOL, (h, g, dev.max())
            worst = max(worst, float(dev.max()))
            s0 = S[u, mem & (ukl == 0)]
            assert s0.size, (h, g, "no level-0 member")
            assert (S[u, ~mem] <= s0.min() - GAP).all(), (h, g, "a non-member is within GAP of level 0")
        anchored(case, h)
    return worst


def anchored(case, h):
    """in every key range (all keys, and each part of the split plan), a group's first tile with members holds a
    level-0 member: the running maximum never moves after a member was summed"""
    ntiles = -(-case.N // TILE)
    for t0, t1 in set(case.ranges) | {(0, ntiles)}:
        for g in range(case.geo.hd):
            ks = case.members(h, g)
            ks = ks[(ks >= TILE * t0) & (ks < TILE * t1)]
            if ks.size:
                first = ks.min() // TILE
                in_first = ks[ks // TILE == first]
                assert (case.klevel[h][in_first] == 0).any(), (h, g, t0, t1, "first member tile has no level 0")


def emulate_p(S):
    """softmax_tile's P for distinct score rows: fp16(2^(s - m + 14)), m the row maximum"""
    return np.exp2(S - S.max(axis=1, keepdims=True) + P_BIAS).astype(np.float16)


def reference(case):
    """(want, terms): fp64 [n N][heads hd] weighted means with the intended weights, and sum(w |v|) / sum(w) of each
    element, the scale of its terms"""
    geo, N = case.geo, case.N
    want = np.zeros((case.n * N, geo.heads * geo.hd))
    terms = np.zeros_like(want)
    for h in range(geo.heads):
        c = slice(h * geo.hd, (h + 1) * geo.hd)
        for b in range(case.n):
            v = case.qkv[b * N:(b + 1) * N, case.cols("v", h)].astype(np.float64)
            for g in range(geo.hd):
                rows = np.nonzero(case.qgroup[h] == g)[0]
                if not rows.size:
                    continue
                mem = case.members(h, g)
                if mem.size:
                    w = 2.0 ** -case.klevel[h][mem].astype(np.float64)
                    mean = w @ v[mem] / w.sum()
                    t = w @ np.abs(v[mem]) / w.sum()
                else:
                    mean, t = v.mean(0), np.abs(v).mean(0)
                want[b * N + rows, c] = mean
                terms[b * N + rows, c] = t
    return want, terms


def error(got, case, want=None, terms=None):
    """max |got - want| relative to the scale of the terms of its row and head, max over the head's dims of
    sum(w |v|) / sum(w).  A per-element scale would measure V's hi + lo split of a tiny value at fp16's subnormal
    spacing instead of the kernel's arithmetic."""
    if want is None:
        want, terms = reference(case)
    hd = case.geo.hd
    scale = terms.reshape(len(terms), -1, hd).max(axis=2, keepdims=True)
    return float((np.abs(got.astype(np.float64) - want).reshape(len(want), -1, hd) / scale).max())
