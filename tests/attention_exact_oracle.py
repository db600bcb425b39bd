"""Element-by-element references for the fused attention kernels (attention.cu K2 forward, K3 backward with its dsum and dQ
finish passes, K4 column sums; attention_export.cu).  Test infrastructure only; no GPU needed.

Layout, as the kernels read it: qkv [B*S, 3H] bf16 with q / k / v of head h at columns h*64 of their block, d_ctx [B*S, H],
scale = 1/8.  A padding query row softmaxes uniformly over all S keys of its sequence (the kernels realise it as zero scores);
its log-sum-exp is ln S and it sends no gradient into q or k.

Routed softmax (routed()).  Every valid query i of (b, h) gets one target key a, or two tied targets a and a ^ 2^t, among the
keys it may see.  Key j of (b, h) carries the +-1 code of the bits of j ^ salt(b, h) in dims [0, nb), 1 in the bias dim, and
in one label dim the poison level X = 4 nb - 2 when some query of the layer must not see it (see LABELS).  The query is
A (code(a)) or A (code(a) + code(b)) plus a bias -A nb or -A (2 nb - 2), and +A in the label dims of every key it must not
see.  With A = 512:
  - the target scores exactly 0, every other admitted key scores <= -2 A (one-hot, one Hamming step) or <= -4 A (two-hot:
    the pair differs in bit t only, so any third key is a further step from the query on the other bits).  In the kernels'
    log2 domain that is <= -2 A (1/8) log2(e) = -184.7, past fp32's normal range: its ex2.approx.ftz is exactly 0.
  - m = 0, so the LSE is 0 (one target) or ln 2 (two), P is exactly 1 or 1/2, and every output is a sum of small dyadic
    rationals.  V, dO are integers in [-1, 1] (padding keys: V = 2; padding query rows: dO = 0), so ctx, D, dV, dS', dK, dQ,
    the bias gradient, the column sums and the export are exact in fp32 and their bf16 roundings are known.
  - one-hot rows have dS = P (dP - D) = 0 exactly (D = dP of the target), so dQ = dK = 0 exactly there; a D read from another
    row or head breaks that.  Two-hot rows have dS = +-(dP_a - dP_b) / 4 on the pair: non-zero and exact.
  - a poisoned key scores >= +2 A if it leaks: it takes all of the probability (K2) or overflows ex2 (K3, K4).  Rows past B*S
    are zero-filled by TMA and score 0: a leak ties with the target and halves it.
  - every tensor-core partial sum is an integer multiple of the operands' granule below 2^16 granules (max_partial_units()).

Counting (counting()).  q = 0: P is uniform over the admitted keys, l = n (the admitted count) and O = sum of V over them, both
exact, so ctx = bf16(fl(O * fl(1/n))) is known bit for bit.  V[j, c] = [j % 32 == c] (c < 32), [(j // 32) % 32 == c - 32]
(c >= 32): no count exceeds 124 < 128, so round(ctx n) recovers every count, and a wrong admitted set names the 32-word
position or word it got wrong.

Random data (reference() with bounds=True).  The float64 reference and, per element, a bound from where the kernels round:
    B9 = 2^-9; one bf16 rounding moves x by at most 2^-8 |x| = 2 B9 |x|.
    ctx:  K2 rounds P to bf16 before the PV MMA (l keeps fp32 P):    (2 B9 + eps2 + 2 gam + 2u) (P|V|) + 1/2 ulp(ctx)
    LSE:  m + log2f(l), times ln 2 (fp32):                              dlse = ln2 ds + eps2 + gam + 4u (|lse| + ln2 T)
    D:    from the bf16 ctx K2 wrote:                                    dD = sum_c |dO| (bar_ctx + ulp(ctx)) + 16u sum |dO ctx|
    dV:   K3 rounds P to bf16 before the dV MMA:                         ((2 B9 + eps3) P)^T |dO| + gam P^T |dO| + 1/2 ulp
    dS':  P (dP - D), rounded to bf16 before the dK / dQ MMAs:           EdS = (2 B9 + eps3 + 2u) G + P (ddP + dD),
          G = P (|dP| + |D|)
    dK:   scale (EdS^T |Q| + gam G^T |Q|) + 1/2 ulp;  dQ: scale (EdS |K| + gam G |K|) + 1/2 ulp  (fp32 slices / red.add and the
          exact x 1/8 are inside gam)
    bias: sum over rows of the dqkv bars + 2 rows u sum |dqkv|
    column sums (fp32 P):  sum_q eps3 P / heads + gam colsum + 2 heads u colsum;   export: sum_h (eps3 + 2^-21) P / heads + ...
  with u = 2^-24, gam = 2 (S + 64) u (an fp32 running sum of <= S + 64 terms, c = 2 for truncating tensor cores),
  T = the row's largest admitted |score| in log2 units, ds = 2 * 64 u QK + 2u T the absolute error of a log2-domain score
  (QK: the row's largest sc2 sum_d |q_d k_d|), eps2 = ln2 (2 ds + 2u T) + 2^-22 the relative error of K2's p (ex2.approx:
  2^-22), eps3 = ln2 (ds + 2u (T + |lse| log2 e)) + dlse + 2^-22 that of P recomputed from the LSE.  Only the 2 B9 terms come
  from bf16; every other term is fp32 rounding and stays below 2^-9 / 4 for S <= 3968 and |scores| <= 64.
"""
from __future__ import annotations

import math

import numpy as np
import torch

FK, AT_N, BQ = 64, 128, 64      # K2 key tile, K3 / K4 key tile, K3 / K4 query chunk
D_HEAD = 64
SCALE = 0.125
A = 512
U = 2.0 ** -24
B9 = 2.0 ** -9
LN2 = math.log(2.0)
LOG2E = 1.0 / LN2
LN2_F32 = float(np.float32(0.6931471805599453))
SC2 = float(np.float32(SCALE) * np.float32(1.4426950408889634))  # p.scale * LOG2E in fp32
MAX_DQ_PARTS = 4
# head dims of the routed construction
BIAS_DIM, PAD_DIM, BATCH_DIM0, LANG_DIM0 = 16, 17, 18, 20   # LANG_DIM0 .. + 6: language labels 3 (b % 2) + chunk % 3
LABELS = "PAD: padding key; BATCH + b % 2: other keys (no pair mask / vision); LANG + 3 (b % 2) + c % 3: language chunk c"


def n_bits(S: int) -> int:
    """Code bits of the routed construction: enough for S keys, and at least 2 so that a poisoned key scores >= +2 A."""
    return max(2, (S - 1).bit_length())


def poison_level(nb: int) -> int:
    return 4 * nb - 2


def dq_parts(S: int) -> int:
    """merlot_attention_bwd_dq_parts: per-key-tile fp32 slices up to 4 key tiles, 0 = one atomically accumulated slice."""
    n = -(-S // AT_N)
    return n if n <= MAX_DQ_PARTS else 0


# ---------------------------------------------------------------------------------------------------------------------
# masks
# ---------------------------------------------------------------------------------------------------------------------
def segments(S: int, pair=(0, 0)) -> torch.Tensor:
    """int64 [S]: 0 for unrestricted positions (vision tokens, or the feature off), 1 + chunk index for language tokens."""
    P, chunk = pair
    t = torch.arange(S)
    if chunk <= 0:
        return torch.zeros(S, dtype=torch.int64)
    return torch.where(t >= P, 1 + (t - P) // chunk, torch.zeros_like(t))


def pair_ok(S: int, pair=(0, 0)) -> torch.Tensor:
    seg = segments(S, pair)
    return (seg[:, None] == seg[None]) | (seg == 0)[:, None] | (seg == 0)[None]


def valid_or_ones(valid, B, S) -> torch.Tensor:
    return torch.ones(B, S, dtype=torch.bool) if valid is None else valid.bool()


def score_mask(valid, B, S, pair=(0, 0)) -> torch.Tensor:
    """bool [B, S, S]: m[q, k] = valid[q] & valid[k] & pair_ok (the reference's mask)."""
    v = valid_or_ones(valid, B, S)
    return v[:, :, None] & v[:, None, :] & pair_ok(S, pair)[None]


def admitted(valid, B, S, pair=(0, 0)) -> torch.Tensor:
    """bool [B, S, S]: the keys each query's softmax runs over (a padding query row: all S keys)."""
    v = valid_or_ones(valid, B, S)
    return score_mask(valid, B, S, pair) | ~v[:, :, None]


def validity(kind: str, B: int, S: int):
    """bool [B, S] or None.  'ragged': lengths S, S - 1, 2S/3 + 1 and holes on 32-position word and tile boundaries in the last
    sequence; 'len1': the first sequence has one token; 'empty': the last sequence is all padding; 'pair': the tail of some
    language chunks is padding (pair_for(S) gives the chunks)."""
    if kind == "none":
        return None
    v = torch.ones(B, S, dtype=torch.bool)
    if kind == "ragged":
        lens = [S, max(1, S - 1), max(1, (2 * S) // 3 + 1)]
        for b in range(B):
            v[b, lens[b % 3]:] = False
        holes = [p for p in (31, 32, 63, 64, 127, 128, 255, 256, 511, 512, 513, 1023, 1024) if p < S - 1]
        if holes:
            v[B - 1, holes] = False
    elif kind == "len1":
        v[0, 1:] = False
    elif kind == "empty":
        v[B - 1] = False
        if B > 1:
            v[0, (3 * S) // 4 + 1:] = False
    elif kind == "pair":
        P, chunk = pair_for(S)
        for c in range(-(-(S - P) // chunk)):
            n_pad = c % 4
            end = min(S, P + (c + 1) * chunk)
            if n_pad and end - n_pad > P + c * chunk:
                v[:, end - n_pad:end] = False
    else:
        raise ValueError(kind)
    return v


def pair_for(S: int):
    """(vision tokens P, chunk length) of disable_pairwise_lang_attn for a sequence of S: chunk boundaries inside 32-position
    words and across 64 / 128-wide tiles."""
    if S < 8:
        return 0, 1
    P = (2 * S) // 5
    chunk = 33 if S > 200 else max(2, S // 5)
    return P, chunk


# ---------------------------------------------------------------------------------------------------------------------
# constructions
# ---------------------------------------------------------------------------------------------------------------------
def _code(x: torch.Tensor, nb: int) -> torch.Tensor:
    """float64 [len(x), nb] of +-1: bit d of x."""
    return ((x[:, None] >> torch.arange(nb)) & 1).double() * 2 - 1


def _labels(B, S, valid, pair):
    """int64 [B, S]: the label dim of every key, and bool [B, S, n_dims] the label dims each query must not see."""
    v = valid_or_ones(valid, B, S)
    seg = segments(S, pair)
    lab = torch.empty(B, S, dtype=torch.int64)
    for b in range(B):
        lab[b] = torch.where(seg > 0, LANG_DIM0 + 3 * (b % 2) + (seg - 1) % 3, torch.full_like(seg, BATCH_DIM0 + b % 2))
    lab[~v] = PAD_DIM
    forbid = torch.zeros(B, S, D_HEAD, dtype=torch.bool)
    forbid[:, :, PAD_DIM] = True
    for b in range(B):
        other = b % 2 ^ 1
        forbid[b, :, BATCH_DIM0 + other] = True
        forbid[b, :, LANG_DIM0 + 3 * other:LANG_DIM0 + 3 * other + 3] = True
        own = LANG_DIM0 + 3 * (b % 2)
        lang_q = seg > 0
        for r in range(3):  # a language query of chunk c sees only its own chunk's language keys
            forbid[b, lang_q & ((seg - 1) % 3 != r), own + r] = True
    return lab, forbid


def routed(B: int, S: int, heads: int, valid=None, pair=(0, 0), seed: int = 0):
    """The routed construction (module docstring).  Returns dict(qkv bf16 [B*S, 3H], d_ctx bf16 [B*S, H], targets int64
    [B, heads, S, 2] (-1: none; padding query rows have none), nb, X)."""
    H = heads * D_HEAD
    g = torch.Generator().manual_seed(seed)
    nb, X = n_bits(S), poison_level(n_bits(S))
    assert nb <= BIAS_DIM
    v = valid_or_ones(valid, B, S)
    adm = score_mask(valid, B, S, pair)
    lab, forbid = _labels(B, S, valid, pair)
    q = torch.zeros(B, S, heads, D_HEAD, dtype=torch.float64)
    k = torch.zeros_like(q)
    vv = torch.randint(-1, 2, (B, S, heads, D_HEAD), generator=g).double()
    vv[~v] = 2.0
    dO = torch.randint(-1, 2, (B, S, heads, D_HEAD), generator=g).double()
    dO[~v] = 0.0
    targets = torch.full((B, heads, S, 2), -1, dtype=torch.int64)
    edges = [S - 1, 63, 64, 127, 128, 31, 32, 0]
    for b in range(B):
        for h in range(heads):
            salt = int(torch.randint(0, 1 << nb, (1,), generator=g))
            idx = torch.arange(S)
            codes = _code(idx ^ salt, nb)
            k[b, :, h, :nb] = codes
            k[b, :, h, BIAS_DIM] = 1.0
            k[b, idx, h, lab[b]] = float(X)
            pick = torch.randint(0, 1 << 30, (S,), generator=g).tolist()
            for i in range(S):
                if not v[b, i]:
                    continue
                keys = adm[b, i].nonzero().flatten()
                n = len(keys)
                r = pick[i]
                a = int(keys[r % n])
                if i % 5 == 0:  # tile and word edges as targets
                    e = edges[(i // 5) % len(edges)]
                    if 0 <= e < S and adm[b, i, e]:
                        a = e
                two = None
                if i % 2 == 1:  # two tied targets a, a ^ 2^t across 32-word, 64- and 128-tile boundaries
                    for t in (5, 6, 7, 0, 1, 4, 8, 9):
                        if t >= nb:
                            continue
                        bb = a ^ (1 << t)
                        if bb < S and adm[b, i, bb]:
                            two = bb
                            break
                targets[b, h, i, 0] = a
                qi = torch.zeros(D_HEAD, dtype=torch.float64)
                if two is None:
                    qi[:nb] = codes[a]
                    qi[BIAS_DIM] = -nb
                else:
                    targets[b, h, i, 1] = two
                    qi[:nb] = codes[a] + codes[two]
                    qi[BIAS_DIM] = -(2 * nb - 2)
                qi[forbid[b, i]] = 1.0
                q[b, i, h] = qi * A
    qkv = torch.stack([q, k, vv], 2).reshape(B * S, 3 * H)
    assert torch.equal(qkv.bfloat16().double(), qkv)
    return dict(qkv=qkv.bfloat16(), d_ctx=dO.reshape(B * S, H).bfloat16(), targets=targets, nb=nb, X=X)


def routed_weights(targets: torch.Tensor, valid, b: int, h: int, S: int) -> torch.Tensor:
    """float64 [S, S] unnormalised weights of (b, h): 1 on the targets of a valid row, 1 on all S keys of a padding row."""
    W = torch.zeros(S, S, dtype=torch.float64)
    t = targets[b, h]
    for c in range(2):
        rows = (t[:, c] >= 0).nonzero().flatten()
        W[rows, t[rows, c]] = 1.0
    if valid is not None:
        W[~valid[b].bool()] = 1.0
    return W


def counting(B: int, S: int, heads: int):
    """The counting construction: q = 0, k = 0, V columns = membership bits (module docstring), d_ctx = 0."""
    H = heads * D_HEAD
    j = torch.arange(S)
    V = torch.zeros(S, D_HEAD, dtype=torch.float64)
    V[j, j % 32] = 1.0
    V[j, 32 + (j // 32) % 32] = 1.0
    qkv = torch.zeros(B, S, 3, heads, D_HEAD, dtype=torch.float64)
    qkv[:, :, 2] = V[None, :, None]
    return dict(qkv=qkv.reshape(B * S, 3 * H).bfloat16(), d_ctx=torch.zeros(B * S, H, dtype=torch.bfloat16))


def random_case(B: int, S: int, heads: int, seed: int, peaked: bool = False):
    """Random bf16 qkv and d_ctx.  peaked: q scaled by 3 and a common direction that the keys of the last 64-key tile share,
    so that most rows take their maximum in the last key tile and K2's online softmax rescales what it has accumulated."""
    H = heads * D_HEAD
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, S, 3, heads, D_HEAD, generator=g)
    if peaked:
        x[:, :, 0] *= 3
        x[:, :, 0, :, 0] = 4.0
        last = ((S - 1) // FK) * FK
        x[:, last:, 1, :, 0] = 6.0
    d_ctx = torch.randn(B * S, H, generator=g) * 0.5
    return x.reshape(B * S, 3 * H).bfloat16(), d_ctx.bfloat16()


def decode_counts(ctx_row: torch.Tensor, n: int) -> torch.Tensor:
    """round(ctx n): the counting construction's per-column counts of admitted keys (exact for counts <= 127)."""
    return (ctx_row.double() * n).round().long()


def max_partial_units(qkv: torch.Tensor, B: int, S: int, heads: int) -> float:
    """Largest sum_d |q_d| |k_d| over all (query, key) pairs of one (b, h), in units of the q granule times the k granule
    (here A x 1): the bound on every partial sum of the score MMAs."""
    H = heads * D_HEAD
    x = qkv.double().reshape(B, S, 3, heads, D_HEAD).abs()
    worst = 0.0
    for b in range(B):
        for h in range(heads):
            worst = max(worst, float((x[b, :, 0, h] @ x[b, :, 1, h].t()).max()) / A)
    return worst


# ---------------------------------------------------------------------------------------------------------------------
# float64 reference, the kernels' exact results on the constructions, and the bounds
# ---------------------------------------------------------------------------------------------------------------------
def _ulp_bf16(x: torch.Tensor) -> torch.Tensor:
    _, e = torch.frexp(x.abs())
    e = torch.where(x == 0, torch.full_like(e, -126), torch.clamp(e - 1, min=-126))
    return torch.ldexp(torch.ones_like(x), e - 7)


def _split_heads(t: torch.Tensor, B, S, heads, blocks):
    return t.double().reshape(B, S, blocks, heads, D_HEAD)


def reference(qkv, d_ctx, B, S, heads, valid=None, pair=(0, 0), *, split=None, weights=None, bounds=False, device="cpu"):
    """float64 outputs of K2 / K3 / K4 / export on qkv, d_ctx (bf16, as the kernels read them).

    weights: None (softmax of the masked scaled scores) or a function (b, h) -> float64 [S, S] unnormalised weights W of an
    exact construction (P = W / rowsum W); then 'ctx_emul' is K2's result bit for bit: bf16(fl(fl(W V) fl(1 / l))).
    split: query index at which the column sums go to the second buffer (None: one buffer).
    Returns a dict of float64 CPU tensors: ctx [B*S, H], lse [B, heads, S], D [B, heads, S], dqkv [B*S, 3H], bias [3H],
    cs[(valid_q, part)] [B, S], export [B, S, S], and with bounds=True the matching 'bar_*' tensors (module docstring;
    the half-ulp output terms are added by the checks)."""
    H = heads * D_HEAD
    dev = torch.device(device)
    x = _split_heads(qkv, B, S, heads, 3).to(dev)
    dO_all = d_ctx.double().reshape(B, S, heads, D_HEAD).to(dev)
    vmask = valid_or_ones(valid, B, S).to(dev)
    m_all = score_mask(valid, B, S, pair).to(dev)
    out = dict(ctx=torch.zeros(B, S, heads, D_HEAD, dtype=torch.float64, device=dev), lse=torch.zeros(B, heads, S, dtype=torch.float64, device=dev),
               D=torch.zeros(B, heads, S, dtype=torch.float64, device=dev),
               dqkv=torch.zeros(B, S, 3, heads, D_HEAD, dtype=torch.float64, device=dev),
               export=torch.zeros(B, S, S, dtype=torch.float64, device=dev))
    cs = {(vq, part): torch.zeros(B, S, dtype=torch.float64, device=dev) for vq in (False, True) for part in (0, 1)}
    if weights is not None:
        out["ctx_emul"] = torch.zeros(B, S, heads, D_HEAD, dtype=torch.bfloat16, device=dev)
    if bounds:
        for name in ("ctx", "lse", "D", "dqkv", "export"):
            out["bar_" + name] = torch.zeros_like(out[name])
        bar_cs = {key: torch.zeros(B, S, dtype=torch.float64, device=dev) for key in cs}
    gam = 2 * (S + 64) * U
    sp = S if split is None else split
    part_of_q = (torch.arange(S, device=dev) >= sp).long()
    for b in range(B):
        vq = vmask[b]
        m = m_all[b]
        adm = m | ~vq[:, None]
        for h in range(heads):
            q, k, v = x[b, :, 0, h], x[b, :, 1, h], x[b, :, 2, h]
            dO = dO_all[b, :, h]
            t = (q @ k.t()) * SCALE
            if weights is None:
                t_eff = torch.where(vq[:, None], torch.where(m, t, torch.full_like(t, -math.inf)), torch.zeros_like(t))
                lse = torch.logsumexp(t_eff, 1)
                P = torch.exp(t_eff - lse[:, None])
            else:
                W = weights(b, h).to(dev)
                l = W.sum(1)
                lse = torch.log(l)
                P = W / l[:, None]
                o = (W @ v).float()
                out["ctx_emul"][b, :, h] = (o * (torch.ones_like(l, dtype=torch.float32) / l.float())[:, None]).bfloat16()
            ctx = P @ v
            dP = dO @ v.t()
            D = (dO * ctx).sum(1)
            gq = vq.double()
            dS = P * (dP - D[:, None]) * gq[:, None]
            out["ctx"][b, :, h] = ctx
            out["lse"][b, h] = lse
            out["D"][b, h] = D
            out["dqkv"][b, :, 0, h] = SCALE * (dS @ k)
            out["dqkv"][b, :, 1, h] = SCALE * (dS.t() @ q)
            out["dqkv"][b, :, 2, h] = P.t() @ dO
            out["export"][b] += P / heads
            for vqf in (False, True):
                sel = gq if vqf else torch.ones_like(gq)
                for part in (0, 1):
                    w = sel * (part_of_q == part).double()
                    cs[(vqf, part)][b] += (w @ P) / heads
            if not bounds:
                continue
            T = torch.where(adm & vq[:, None], t.abs() * LOG2E, torch.zeros_like(t)).amax(1)
            QK = torch.where(adm & vq[:, None], (q.abs() @ k.abs().t()) * SC2, torch.zeros_like(t)).amax(1)
            ds = 2 * 64 * U * QK + 2 * U * T
            eps2 = LN2 * (2 * ds + 2 * U * T) + 2.0 ** -22
            dlse = LN2 * ds + eps2 + gam + 4 * U * (lse.abs() + LN2 * T)
            eps3 = LN2 * (ds + 2 * U * (T + lse.abs() * LOG2E)) + dlse + 2.0 ** -22
            bar_ctx = (2 * B9 + eps2[:, None] + 2 * gam + 2 * U) * (P @ v.abs())
            dD = (dO.abs() * (bar_ctx + _ulp_bf16(ctx))).sum(1) + 16 * U * (dO * ctx).abs().sum(1)
            ddP = 2 * 64 * U * (dO.abs() @ v.abs().t())
            G = P * (dP.abs() + D.abs()[:, None]) * gq[:, None]
            EdS = (2 * B9 + eps3[:, None] + 2 * U) * G + P * (ddP + dD[:, None]) * gq[:, None]
            out["bar_ctx"][b, :, h] = bar_ctx
            out["bar_lse"][b, h] = dlse
            out["bar_D"][b, h] = dD
            out["bar_dqkv"][b, :, 0, h] = SCALE * (EdS @ k.abs() + gam * (G @ k.abs()))
            out["bar_dqkv"][b, :, 1, h] = SCALE * (EdS.t() @ q.abs() + gam * (G.t() @ q.abs()))
            out["bar_dqkv"][b, :, 2, h] = ((2 * B9 + eps3[:, None]) * P).t() @ dO.abs() + gam * (P.t() @ dO.abs())
            out["bar_export"][b] += (eps3[:, None] + 2.0 ** -21) * P / heads
            for vqf in (False, True):
                sel = gq if vqf else torch.ones_like(gq)
                for part in (0, 1):
                    w = sel * (part_of_q == part).double()
                    bar_cs[(vqf, part)][b] += ((w * eps3) @ P + gam * (w @ P)) / heads
    res = {key: val.cpu() for key, val in out.items()}
    res["ctx"] = res["ctx"].reshape(B * S, H)
    res["dqkv"] = res["dqkv"].reshape(B * S, 3 * H)
    res["bias"] = res["dqkv"].sum(0)
    res["cs"] = {key: val.cpu() for key, val in cs.items()}
    if weights is not None:
        res["ctx_emul"] = res["ctx_emul"].reshape(B * S, H)
    if bounds:
        res["bar_ctx"] = res["bar_ctx"].reshape(B * S, H)
        res["bar_dqkv"] = res["bar_dqkv"].reshape(B * S, 3 * H)
        res["bar_export"] = res["bar_export"] + 2 * U * heads * res["export"]
        res["bar_cs"] = {key: val.cpu() + 2 * U * heads * res["cs"][key] for key, val in bar_cs.items()}
        half = 0.5 * _ulp_bf16(res["dqkv"].abs() * (1 + 2.0 ** -7))
        res["bar_bias"] = (res["bar_dqkv"] + half).sum(0) + 2 * B * S * U * res["dqkv"].abs().sum(0)
    return res


# ---------------------------------------------------------------------------------------------------------------------
# where an element sits, and the checks
# ---------------------------------------------------------------------------------------------------------------------
def where_qkv(kind: str, B: int, S: int, heads: int, row: int, col: int) -> str:
    """'(b, h, row, col)' plus the tile and chunk the element belongs to, for a [B*S, width] tensor (kind: 'query' rows
    (ctx, dq: K2 query tile of 128, K3 query chunk of 64, 32-word) or 'key' rows (dk, dv: K2 key tile of 64, K3 key tile
    of 128))."""
    b, i = divmod(row, S)
    h, c = divmod(col % (heads * D_HEAD), D_HEAD)
    if kind == "query":
        loc = f"K2 query tile {i // 128}, K3/K4 query chunk {i // BQ}, word {i // 32}"
    else:
        loc = f"K2 key tile {i // FK}, K3/K4 key tile {i // AT_N}, word {i // 32}"
    return f"(b={b}, h={h}, row={i}, col={c}) [{loc}]"


def where_bhs(B, S, heads, idx) -> str:
    b, h, i = idx
    return f"(b={b}, h={h}, row={i}) [K2 query tile {i // 128}, K3/K4 query chunk {i // BQ}, word {i // 32}]"


def bound_check(got, ref, bar, what, locate, *, out_bf16=True):
    """|got - ref| <= bar (+ 1/2 bf16 ulp of max(|got|, |ref|) for a bf16 output), element by element.  locate(index tuple)
    names the element.  Returns the worst err / bound."""
    got = got.detach().to(torch.float64).cpu()
    ref, bar = ref.to(torch.float64), bar.to(torch.float64)
    bad = ~torch.isfinite(got)
    if bool(bad.any()):
        idx = tuple(int(j) for j in bad.nonzero()[0])
        raise AssertionError(f"{what}: {int(bad.sum())} non-finite elements, first at {locate(idx)}: {float(got[idx])!r}")
    bound = bar
    if out_bf16:
        bound = bound + 0.5 * _ulp_bf16(torch.maximum(got.abs(), ref.abs()))
    bound = bound.clamp(min=2.0 ** -149)
    ratio = (got - ref).abs() / bound
    i = int(ratio.argmax())
    idx = tuple(int(j) for j in np.unravel_index(i, tuple(ratio.shape)))
    worst = float(ratio.reshape(-1)[i])
    assert worst <= 1.0, (f"{what}: element {locate(idx)}: got {float(got[idx])!r}, float64 {float(ref[idx])!r}, {worst:.3g} x "
                          f"the bound {float(bound[idx]):.3g}")
    return worst


def exact_check(got, want, what, locate):
    """Bitwise equality (torch.equal) naming the first wrong element and how many there are."""
    got = got.detach().cpu()
    assert got.shape == want.shape and got.dtype == want.dtype, (what, got.shape, got.dtype, want.shape, want.dtype)
    if torch.equal(got, want):
        return
    bad = got.ne(want) | (got.isnan() if got.is_floating_point() else torch.zeros_like(got, dtype=torch.bool))
    n = int(bad.sum())
    idx = tuple(int(j) for j in bad.nonzero()[0])
    raise AssertionError(f"{what}: {n} of {got.numel()} elements differ; first at {locate(idx)}: got {float(got[idx])!r}, "
                         f"want {float(want[idx])!r}")


def ulp_check(got, want, ulps, what, locate):
    """|got - want| <= ulps * ulp_f32(want) element by element (fp32 sums of fp32 terms in an unspecified order)."""
    got = got.detach().double().cpu()
    want = want.double()
    _, e = torch.frexp(want.abs())
    e = torch.where(want == 0, torch.full_like(e, -126), torch.clamp(e - 1, min=-126))
    u = torch.ldexp(torch.ones_like(want), e - 23)
    err = (got - want).abs()
    bad = ~(err <= ulps * u)
    if bool(bad.any()):
        idx = tuple(int(j) for j in bad.nonzero()[0])
        raise AssertionError(f"{what}: {int(bad.sum())} elements beyond {ulps} ulps; first at {locate(idx)}: got "
                             f"{float(got[idx])!r}, want {float(want[idx])!r}")


# ---------------------------------------------------------------------------------------------------------------------
# float32 emulation of the kernels' rounding points (CPU)
# ---------------------------------------------------------------------------------------------------------------------
def emulate_fp32(qkv, d_ctx, B, S, heads, valid=None, pair=(0, 0)):
    """The kernels' arithmetic in float32 on the CPU, one rounding point at a time: K2 runs the online softmax over 64-key
    tiles in the log2 domain with bf16 P into the PV product and fp32 P into l; ctx and the LSE as K2 writes them; D from
    the bf16 ctx; K3 recomputes P from the LSE, rounds P to bf16 for dV and dS' = P (dP - D) to bf16 for dK and dQ; dQ is
    scaled by 1/8 after the sum; K4 sums fp32 P.  exp2 is exact here (the GPU's ex2.approx is within 2^-22)."""
    H = heads * D_HEAD
    f32 = torch.float32
    x = qkv.float().reshape(B, S, 3, heads, D_HEAD)
    dO_all = d_ctx.float().reshape(B, S, heads, D_HEAD)
    vmask = valid_or_ones(valid, B, S)
    m_all = score_mask(valid, B, S, pair)
    ctx_o = torch.zeros(B, S, heads, D_HEAD, dtype=torch.bfloat16)
    lse_o = torch.zeros(B, heads, S, dtype=f32)
    D_o = torch.zeros(B, heads, S, dtype=f32)
    dqkv = torch.zeros(B, S, 3, heads, D_HEAD, dtype=torch.bfloat16)
    cs = torch.zeros(B, S, dtype=f32)
    sc2 = torch.tensor(SC2, dtype=f32)
    for b in range(B):
        vq, m = vmask[b], m_all[b]
        for h in range(heads):
            q, k, v = x[b, :, 0, h], x[b, :, 1, h], x[b, :, 2, h]
            dO = dO_all[b, :, h]
            s = (q @ k.t()) * sc2
            t = torch.where(vq[:, None], torch.where(m, s, torch.full_like(s, -1e10 * 1.4426950408889634)), torch.zeros_like(s))
            mr = torch.full((S,), -math.inf, dtype=f32)
            lr = torch.zeros(S, dtype=f32)
            o = torch.zeros(S, D_HEAD, dtype=f32)
            for j0 in range(0, S, FK):
                tj = t[:, j0:j0 + FK]
                mn = torch.maximum(mr, tj.amax(1))
                fct = torch.exp2(mr - mn)
                p = torch.exp2(tj - mn[:, None])
                lr = lr * fct + p.sum(1)
                o = o * fct[:, None] + p.bfloat16().float() @ v[j0:j0 + FK]
                mr = mn
            ctx = (o * (1.0 / lr)[:, None]).bfloat16()
            lse = ((mr + torch.log2(lr)) * torch.tensor(LN2_F32, dtype=f32))
            ctx_o[b, :, h], lse_o[b, h] = ctx, lse
            D = (dO * ctx.float()).sum(1)
            D_o[b, h] = D
            nl = -lse * torch.tensor(1.4426950408889634, dtype=f32)
            pr = torch.exp2(t + nl[:, None])
            dp = dO @ v.t()
            dsv = ((dp - D[:, None]) * torch.where(vq[:, None], pr, torch.zeros_like(pr))).bfloat16().float()
            dqkv[b, :, 0, h] = ((dsv @ k) * SCALE).bfloat16()
            dqkv[b, :, 1, h] = ((dsv.t() @ q) * SCALE).bfloat16()
            dqkv[b, :, 2, h] = (pr.bfloat16().float().t() @ dO).bfloat16()
            cs[b] += pr.sum(0) / heads
    return dict(ctx=ctx_o.reshape(B * S, H), lse=lse_o, D=D_o, dqkv=dqkv.reshape(B * S, 3 * H), cs=cs)
