"""Attention inputs whose every score is set by construction, and a float64 model of the online-softmax schedule of
`flash_kernel` (fgt_b200/csrc/flash.cu). Shared by tests/test_attention_softmax.py (CPU: every case takes the branches
its name promises, and the model is the softmax) and tests/test_attention_softmax_gpu.py (the kernel against the float64
interpreter, with a per-element bar from the model).

Construction. Query row r of head h is the basis vector e_(r mod 128) of that head, so its score with key k is the one
element K[k, h * 128 + r mod 128]: a single product, exact in fp32 in the split-bf16 and in the fp16 build. Every Q, K
and V element is a bf16 value (8 significant bits) that is zero or inside fp16's normal range, so the lo planes are zero
and the fp16 operands hold the same numbers: the float64 softmax of the operands is the exact result, and what remains
under test is the schedule, ex2.approx, P's 16-bit rounding and the fp32 accumulations. Scores are designed in log2
units x = S c, c = fp32(fp32(scale) * fp32(log2 e)) as the kernel forms it. At FGT's scale 1/sqrt(128) the designed x
are rounded through bf16 S, so steps land within a few hundredths of their target; at EXACT_SCALE (about 0.173) c is
exactly 1/4 and integer x are exact, so a step of 8.0 sits exactly on the rescale threshold and every P is a power of 2.

The schedule (flash.cu, restated): the keys of a row are consumed in 64-key tiles, dense in key order, windowed as the
pooled tiles and then the row's own window tile (the other warpgroup's window tile is skipped). Per row, with the tile's
largest live score m_tile = fp32(max S * c) and a reference maximum m_ref (initially -inf): when m_tile > m_ref + 8
(fp32), alpha = 2^(m_ref - m_tile), m_ref = m_tile, and l_run and o are multiplied by alpha; then P = 2^(S c - m_ref)
(fma, ex2.approx with subnormal results flushed to 0; masked columns 0), l_run += sum P in fp32 and o += P16 V with P16
P's 16-bit form (hi + lo of split-bf16, or fp16 with saturation). The output is o / l_run.
"""
import dataclasses
import math

import torch

F64 = torch.float64
LOG2E32 = torch.tensor(1.4426950408889634, dtype=torch.float32)
FGT_SCALE = 1.0 / math.sqrt(128)
THRESHOLD = 8.0
FLUSH = -126.0   # ex2.approx.ftz: 2^t below the smallest normal fp32 is 0


def c32(scale):
    """The kernel's scale_log2 as a float32 tensor."""
    return torch.tensor(scale, dtype=torch.float32) * LOG2E32


def _exact_scale():
    s = torch.tensor(0.25 / 1.4426950408889634, dtype=torch.float32)
    for _ in range(8):
        c = float(c32(s.item()))
        if c == 0.25:
            return s.item()
        s = torch.nextafter(s, torch.tensor(math.inf if c < 0.25 else -math.inf, dtype=torch.float32))
    raise AssertionError("no fp32 scale gives scale_log2 == 1/4")


EXACT_SCALE = _exact_scale()


def r16(x):
    """Nearest bf16 value as float64, zero below 2^-6 in magnitude: held exactly by bf16 (lo plane 0) and by fp16."""
    y = torch.as_tensor(x, dtype=F64).to(torch.bfloat16).double()
    y = torch.where(y.abs() < 2.0 ** -6, torch.zeros_like(y), y)
    assert bool((y.abs() <= 65504).all()), "score or value outside fp16's range"
    return y


@dataclasses.dataclass
class Case:
    name: str
    mode: int           # 0 dense, 1 windowed
    B: int
    H: int
    Lq: int
    Lk: int
    R: int              # Lk_rows
    G: int              # windowed: pooled keys [Lq, Lq + G)
    scale: float
    q: torch.Tensor     # [B, Lq, H * 128] float64 (bf16- and fp16-exact)
    k: torch.Tensor     # [B, R, H * 128]
    v: torch.Tensor     # [B, R, H * 128]
    rowmap: torch.Tensor  # int32 [B * Lq]: output row, -1 dropped
    rows_out: int
    intent: dict

    @property
    def C(self):
        return self.H * 128

    def groups(self):
        """(b, h, query rows, key index [T, 64], live [T, 64]) per run of rows that share one key sequence, tiles in
        the kernel's order. Key indices >= R read as zero rows (TMA fills outside the addressable rows with zeros)."""
        col = torch.arange(64)
        for b in range(self.B):
            for h in range(self.H):
                if self.mode == 0:
                    T = -(-self.Lk // 64)
                    kidx = torch.arange(T)[:, None] * 64 + col
                    yield b, h, torch.arange(self.Lq), kidx, kidx < self.Lk
                    continue
                Tg = -(-self.G // 64)
                gl = torch.arange(Tg)[:, None] * 64 + col
                for qt in range(self.Lq // 128):
                    for wg in range(2):
                        own = (2 * qt + wg) * 64 + col
                        kidx = torch.cat([self.Lq + gl, own[None]])
                        live = torch.cat([gl < self.G, torch.ones(1, 64, dtype=torch.bool)])
                        yield b, h, qt * 128 + wg * 64 + torch.arange(64), kidx, live

    def loaded(self, b, h, rows, kidx):
        """(scores [rows, T, 64] as a tile holds them, float32; values [T, 64, 128] float64) of one group."""
        cols = slice(h * 128, h * 128 + 128)
        inside = kidx < self.R
        kk = torch.zeros(*kidx.shape, 128, dtype=F64)
        vv = torch.zeros(*kidx.shape, 128, dtype=F64)
        kk[inside] = self.k[b, kidx[inside], cols]
        vv[inside] = self.v[b, kidx[inside], cols]
        s = torch.einsum("rd,tkd->rtk", self.q[b, rows, cols], kk)
        return s.float(), vv

    def launch_kwargs(self):
        C = self.C
        kw = dict(batches=self.B, heads=self.H, Lq=self.Lq, Lk=self.Lk, Lk_rows=self.R, q_ld=C, k_ld=C, v_ld=C,
                  out_ld=C, q_batch_stride=self.Lq * C, k_batch_stride=self.R * C, v_batch_stride=self.R * C,
                  out_batch_stride=self.Lq * C, scale=self.scale, mode=self.mode)
        if self.mode == 1:
            kw.update(glob_start=self.Lq, glob_count=self.G)
        return kw


# ------------------------------------------------------------------------------------------------------- the model
@dataclasses.dataclass
class Schedule:
    grow: torch.Tensor      # [rows, T] rescale taken at tile t (the first finite maximum included)
    m_ref: torch.Tensor     # [rows, T] fp32 reference maximum after tile t
    alpha: torch.Tensor     # [rows, T]
    pmax: torch.Tensor      # [rows, T] largest P of tile t (float64, before its 16-bit rounding)
    p16max: torch.Tensor    # [rows, T] largest P16
    l_run: torch.Tensor     # [rows]
    out: torch.Tensor = None   # [rows, 128] o / l_run
    err: torch.Tensor = None   # [rows, 128] sum (P eps + |P16 - P|) |V| / l_run
    mag: torch.Tensor = None   # [rows, 128] sum P |V| / l_run
    rel: torch.Tensor = None   # [rows] sum P eps / l_run

    def rescales_after_first(self):
        """Rescales per row after the one that takes the first finite maximum."""
        return (self.grow.sum(1) - 1).clamp_min(0)


def ex2(t):
    """ex2.approx.ftz modelled exactly: 2^t, 0 below the smallest normal fp32."""
    t = t.double()
    return torch.where(t < FLUSH, torch.zeros_like(t), torch.exp2(t))


def round_p(p, f16):
    """P's 16-bit form: fp32 P split into bf16 hi + lo, or fp16 (round to nearest, saturating at 65504)."""
    p32 = p.float()
    if f16:
        return p32.clamp(max=65504.0).half().double()
    hi = p32.bfloat16().float()
    return hi.double() + (p32 - hi).bfloat16().double()


def schedule(s, live, scale, f16=None, v=None):
    """The schedule on scores s [rows, T, 64] (float32, as loaded) with live columns live [T, 64]. f16: None keeps P
    unrounded, else P16 = round_p(P, f16). With values v [T, 64, D] also the output and the bar parts."""
    c = c32(scale)
    rows, T, _ = s.shape
    masked = torch.where(live, s, torch.tensor(-math.inf))
    m_tile = masked.amax(-1) * c                       # fp32 product, one rounding, as quad_max(mx) * scale_log2
    m = torch.full((rows,), -math.inf, dtype=torch.float32)
    grow = torch.zeros(rows, T, dtype=torch.bool)
    m_ref = torch.empty(rows, T, dtype=torch.float32)
    alpha = torch.ones(rows, T, dtype=F64)
    for t in range(T):
        gr = m_tile[:, t] > m + THRESHOLD
        alpha[:, t] = torch.where(gr, ex2(m - m_tile[:, t]), torch.ones(rows, dtype=F64))
        m = torch.where(gr, m_tile[:, t], m)
        grow[:, t], m_ref[:, t] = gr, m
    neg_m = torch.where(m_ref == -math.inf, torch.zeros_like(m_ref), -m_ref)
    x = s.double() * c.double()
    texp = (x + neg_m.double()[..., None]).float()     # fmaf(s, scale_log2, -m_ref): one rounding to fp32
    p = torch.where(live, ex2(texp), torch.zeros((), dtype=F64))
    p16 = p if f16 is None else round_p(p, f16)
    sch = Schedule(grow, m_ref, alpha, p.amax(-1), p16.amax(-1), torch.zeros(rows, dtype=F64))
    l_run = torch.zeros(rows, dtype=F64)
    for t in range(T):
        l_run = l_run * alpha[:, t] + p[:, t].sum(-1)
    sch.l_run = l_run
    if v is None:
        return sch
    # per key relative weight error: ex2.approx (2^-22) and the fp32 roundings of the exponent (c, the fma, m_tile,
    # each rescale's m_ref - m_tile), at most 2^-24 ln2 times |exponent| each, the exponent bounded by the key's
    # distance below the final reference maximum plus the 8 of the threshold
    eps = 2.0 ** -21 + 2.0 ** -22 * ((m_ref[:, -1:, None].double() - x).clamp_min(0) + 16.0)
    o = torch.zeros(rows, v.shape[-1], dtype=F64)
    err, mag, rel = torch.zeros_like(o), torch.zeros_like(o), torch.zeros(rows, dtype=F64)
    av = v.abs()
    for t in range(T):
        a = alpha[:, t]
        o = o * a[:, None] + p16[:, t] @ v[t]
        err = err * a[:, None] + (p[:, t] * eps[:, t] + (p16[:, t] - p[:, t]).abs()) @ av[t]
        mag = mag * a[:, None] + p[:, t] @ av[t]
        rel = rel * a + (p[:, t] * eps[:, t]).sum(-1)
    sch.out, sch.err, sch.mag, sch.rel = o / l_run[:, None], err / l_run[:, None], mag / l_run[:, None], rel / l_run
    return sch


def softmax_rows(case, b, h, rows, kidx, live):
    """float64 softmax(S * scale) V of one group over its live keys (the operands are exact, so this is the result)."""
    s, v = case.loaded(b, h, rows, kidx)
    sc = torch.tensor(case.scale, dtype=torch.float32).item()
    w = torch.softmax(torch.where(live, s.double() * sc, torch.tensor(-math.inf, dtype=F64)).flatten(1), -1)
    return w @ v.flatten(0, 1)


# --------------------------------------------------------------------------------------------------------- cases
def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _values(B, R, C, g):
    """V over the whole fp16-exact range: 8-bit mantissas times 2^-6 .. 2^8 (so up to +-65280), a fifth of them at
    +-(61440 .. 65280)."""
    mant = torch.randint(-255, 256, (B, R, C), generator=g).double()
    ex = torch.randint(-6, 9, (B, R, C), generator=g).double()
    v = mant * torch.exp2(ex)
    big = torch.rand(B, R, C, generator=g) < 0.2
    top = (torch.randint(240, 256, (B, R, C), generator=g) * 256).double() * torch.sign(mant + 0.5)
    return r16(torch.where(big, top, v))


def _spread(n_rows, T, live_per_tile, g, integer):
    """[n_rows, T, 64] distances below the tile maximum: 0 at one live column of every tile, 1 .. 7 elsewhere
    (integers at EXACT_SCALE, so every P stays a power of 2)."""
    if integer:
        d = torch.randint(1, 8, (n_rows, T, 64), generator=g).double()
    else:
        d = 1.0 + 6.0 * torch.rand(n_rows, T, 64, generator=g, dtype=F64)
    top = (torch.rand(n_rows, T, generator=g, dtype=F64) * live_per_tile.double()).long()
    return d.scatter(2, top[..., None], 0.0)


def _make(name, x_of, *, mode=0, B=2, H=2, Lq, Lk, R=None, G=0, scale=FGT_SCALE, seed, intent):
    """Case whose head-h scores of batch b are x_of(b, h, g) [128, R] in log2 units (row = query direction)."""
    R = Lk if R is None else R
    C = H * 128
    g = _gen(seed)
    c = float(c32(scale))
    k = torch.zeros(B, R, C, dtype=F64)
    for b in range(B):
        for h in range(H):
            k[b, :, h * 128:(h + 1) * 128] = r16(x_of(b, h, g) / c).t()
    q = torch.zeros(B, Lq, C, dtype=F64)
    r = torch.arange(Lq)
    for h in range(H):
        q[:, r, h * 128 + r % 128] = 1.0
    v = _values(B, R, C, g)
    rows_out = B * Lq + 9
    rowmap = torch.randperm(rows_out, generator=g)[:B * Lq].to(torch.int32)
    rowmap[::7] = -1
    return Case(name, mode, B, H, Lq, Lk, R, G, scale, q, k, v, rowmap, rows_out, intent)


def _dense(name, tile_max, *, Lk, R=None, Lq=200, scale=FGT_SCALE, seed, intent, after=None):
    """Dense case: tile t of direction i has its maximum tile_max(b, h)[i, t] (log2 units) at one live column, the
    other keys 1-7 below; after(b, h, x) may overwrite keys (e.g. rows past Lk)."""
    T = -(-Lk // 64)
    live = (Lk - 64 * torch.arange(T)).clamp(max=64)
    R = Lk if R is None else R

    def x_of(b, h, g):
        x = tile_max(b, h)[:, :, None] - _spread(128, T, live, g, scale == EXACT_SCALE)
        x = x.reshape(128, T * 64)
        full = torch.zeros(128, max(R, T * 64), dtype=F64)
        full[:, :T * 64] = x
        full = full[:, :R]
        return after(b, h, full) if after else full
    return _make(name, x_of, Lq=Lq, Lk=Lk, R=R, scale=scale, seed=seed, intent=intent)


def _rise(delta, scale=FGT_SCALE, seed=0):
    T = 6
    shift = lambda b, h: 3.0 * b - 2.0 * h   # noqa: E731  (softmax-invariant, moves m_ref)
    # centred on 0, so that the bf16 scores keep a step at FGT's scale within 0.07 of delta
    tm = lambda b, h: ((torch.arange(T, dtype=F64) - (T - 1) / 2) * delta + shift(b, h)).expand(128, T)   # noqa: E731
    tag = "exact" if scale == EXACT_SCALE else "fgt"
    return _dense(f"rise{delta:g}_{tag}", tm, Lk=T * 64, scale=scale, seed=100 + seed,
                  intent=dict(kind="rise", delta=delta, tiles=T))


def _fall():
    T = 6
    tm = lambda b, h: (-40.0 * torch.arange(T, dtype=F64) + b).expand(128, T)   # noqa: E731
    return _dense("fall40", tm, Lk=T * 64 - 9, seed=200, intent=dict(kind="fall", tiles=T))


def _constant():
    Lk = 21000
    return _make("constant21k", lambda b, h, g: torch.zeros(128, Lk, dtype=F64), B=2, H=2, Lq=130, Lk=Lk, seed=300,
                 intent=dict(kind="constant"))


RESCALE_TILES = {(0, 0): (2, 4), (0, 1): (1, 3, 5), (1, 0): (1, 5), (1, 1): (3,)}   # (warpgroup, half) -> tiles


def _rows_differ():
    """Rows g and g + 8 of a quad pair, and warpgroups 0 and 1, rise by 12 (log2) at different tiles; in between the
    tile maxima sit 2 below the current level."""
    T = 6

    def tm(b, h):
        out = torch.empty(128, T, dtype=F64)
        for i in range(128):
            at = RESCALE_TILES[(i // 64, (i % 16) // 8)]
            lvl = 0.0
            for t in range(T):
                if t in at:
                    lvl += 12.0
                out[i, t] = lvl - (0.0 if t in at or t == 0 else 2.0)
        return out + b - h
    return _dense("rows_differ", tm, Lk=T * 64, Lq=300, scale=EXACT_SCALE, seed=400,
                  intent=dict(kind="rows_differ", tiles=T))


def _partial(rem, inside):
    """Last key tile with `rem` live columns; its live maximum rises by 10 (a rescale on the partial tile). inside: the
    keys right after Lk lie inside Lk_rows and dominate by 50; otherwise Lk_rows = Lk and every live score is at most
    -45, so the columns past the buffer, which TMA fills with zero keys (score 0), dominate."""
    T = 6
    Lk = 64 * (T - 1) + rem
    R = Lk + (7 if inside and rem < 63 else 1 if inside else 0)
    base = 0.0 if inside else -60.0

    def tm(b, h):
        return (torch.tensor([0.0, 3.0, 1.0, 5.0, 2.0, 15.0], dtype=F64) + base).expand(128, T)

    def after(b, h, x):
        if inside:
            x[:, Lk:] = x[:, :Lk].amax(1, keepdim=True) + 50.0
        return x
    return _dense(f"partial{rem}_{'inside' if inside else 'past'}", tm, Lk=Lk, R=R, Lq=70 + rem, seed=500 + rem,
                  intent=dict(kind="partial", rem=rem, inside=inside, tiles=T), after=after)


def _windowed(G, own=20.0):
    """Windowed: 4 windows of 64 queries, G pooled keys whose tiles rise by 9, the own window `own` above the last
    pooled maximum (the rescale on the last tile), the other warpgroup's window tile 80 above everything and the
    padding rows after the pooled keys 60 above."""
    Lq = 256
    Tg = -(-G // 64)
    R = Lq + Tg * 64 + 8

    def x_of(b, h, g):
        x = torch.empty(128, R, dtype=F64)
        glive = (G - 64 * torch.arange(Tg)).clamp(max=64)
        gx = (9.0 * torch.arange(Tg, dtype=F64))[None, :, None] - _spread(128, Tg, glive, g, False)
        x[:, Lq:Lq + Tg * 64] = gx.reshape(128, -1) + b
        top = 9.0 * (Tg - 1) + b
        lx = top + own - _spread(128, Lq // 64, torch.full((Lq // 64,), 64), g, False).reshape(128, Lq)
        mine = (torch.arange(Lq)[None, :] // 64) % 2 == (torch.arange(128)[:, None] // 64)
        x[:, :Lq] = torch.where(mine, lx, top + 80.0)
        x[:, Lq + G:] = top + 60.0
        return x
    return _make(f"windowed_g{G}", x_of, mode=1, Lq=Lq, Lk=R, R=R, G=G, seed=600 + G,
                 intent=dict(kind="windowed", glob_tiles=Tg))


def all_cases():
    return ([_rise(d) for d in (7.9, 8.0, 8.1, 16.0, 40.0, 140.0)] +
            [_rise(8.0, EXACT_SCALE, 1), _rise(16.0, EXACT_SCALE, 2), _fall(), _constant(), _rows_differ()] +
            [_partial(rem, inside) for rem in (1, 63) for inside in (True, False)] +
            [_windowed(65), _windowed(127)])


def schedules(case, f16):
    """[(b, h, rows, Schedule with values)] of every group of the case."""
    out = []
    for b, h, rows, kidx, live in case.groups():
        s, v = case.loaded(b, h, rows, kidx)
        out.append((b, h, rows, schedule(s, live, case.scale, f16, v)))
    return out
