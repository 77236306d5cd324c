"""fp64 attention references and the per-element bound the attention kernels are held to (head-dim-128 prefill attention in
test_gpu_qwen_kernels.py and test_gpu_attention_d128.py, head-dim-64 attention in test_gpu_attention_d64.py), the kernels' exponent
reference, row sampling for long sequences, and the key-code selector fixtures of the head-dim-128 and flash-decoding kernels."""
import torch


def bf16_ulp(x):
    """Spacing of bf16 at |x| (8 significant bits)."""
    a = x.abs().double().clamp_min(2.0 ** -126)
    return torch.exp2(torch.floor(torch.log2(a)) - 7)


def softmax_ref(s, v, m=None):
    """softmax(s) v in fp64 for scores s [..., n, m] (natural-log domain, -inf where masked; every row has a finite score) and v [..., m, d].
    Returns (exact, the same with P = exp(s - m) rounded to bf16 before P.V and l summed unrounded): the kernels' one deliberate rounding.
    m [..., n, 1]: the exponent reference the kernel rounds P at, within 8 ln 2 below the row maximum; default the row maximum."""
    e = torch.exp(s - (s.amax(-1, keepdim=True) if m is None else m))
    l = e.sum(-1, keepdim=True)
    v = v.double()
    return torch.matmul(e, v) / l, torch.matmul(e.to(torch.bfloat16).double(), v) / l


def attn_ref(q, k, v, scale, causal, q_off=0):
    """fp64 attention of q [H, n, d] over k, v [H, m, d]; query i sits at key position i + q_off (causal: sees keys j <= i + q_off).
    Returns softmax_ref's pair (exact, P rounded to bf16)."""
    q, k = q.double(), k.double()
    s = torch.matmul(q, k.transpose(1, 2)) * scale
    if causal:
        i = torch.arange(q.shape[1], device=q.device)[:, None] + q_off
        j = torch.arange(k.shape[1], device=q.device)[None, :]
        s = s.masked_fill(j > i, float("-inf"))
    return softmax_ref(s, v)


def attn_bound(ref, ref_p):
    """Per element: one bf16 ulp of the output plus 2x the largest error of the P-rounding restatement in that head (the kernel rounds P at
    its own exponent reference, so its rounding errors are another draw of the same size, not the same errors)."""
    return bf16_ulp(ref) + 2.0 * (ref_p - ref).abs().amax((-2, -1), keepdim=True)


def assert_attn(got, ref, ref_p, what):
    assert bool(torch.isfinite(got).all()), f"{what}: non-finite output"
    tol = attn_bound(ref, ref_p)
    excess = (got.double() - ref).abs() - tol
    assert float(excess.max()) <= 0.0, f"{what}: {int((excess > 0).sum())} elements past the bound, worst by {float(excess.max()):.3g}"
    return tol


def assert_discriminates(wrong, ref, tol, what, factor=4.0):
    """A plausible kernel mistake, applied to the reference, must move some element by `factor` x the tolerance."""
    assert bool(((wrong - ref).abs() > factor * tol).any()), f"fixture cannot see {what}"


LN2 = 0.6931471805599453


def exponent_reference(s):
    """The kernel's exponent reference of each row: the maximum of its first 128-key tile, raised to a later tile's maximum only when that
    exceeds it by more than 2^8 (8 ln 2 here, in the natural-log domain). A row dominated by one key then rounds that key's P as the kernel
    does, not to an exact 1."""
    tiles = [s[..., t:t + 128].amax(-1, keepdim=True) for t in range(0, s.shape[-1], 128)]
    m = tiles[0]
    for t in tiles[1:]:
        m = torch.where(t > m + 8 * LN2, t, m)
    return m


def masked_ref(q, k, v, scale, visible):
    """fp64 attention of q [H, n, d] over k, v [H, m, d] with visible [n, m] (or [H, n, m]) bool, P rounded at the kernel's exponent
    reference: key column c of the arrays must sit at column c mod 128 of the kernel's key tile c // 128 (pad with invisible columns where
    the kernel's tiles restart, as after a shared prefix). Returns softmax_ref's pair."""
    s = torch.matmul(q.double(), k.double().transpose(-1, -2)) * scale
    s = s.masked_fill(~visible, float("-inf"))
    return softmax_ref(s, v, exponent_reference(s))


def sample_row_blocks(n, block=1024, spread=4):
    """Query-row blocks [r0, r1) to check of an n-row sequence: every block up to (spread + 2) blocks, otherwise the first block, the last
    one (it holds the ragged last query tile) and `spread` evenly spaced blocks between them, all starting on 128-row tiles. Bounds the fp64
    score memory (block x keys x 8 bytes per head) and the time of long sequences."""
    starts = list(range(0, n, block))
    if len(starts) > spread + 2:
        last = max(0, (n - block + 127) // 128 * 128)
        mid = [int(round(x)) // 128 * 128 for x in torch.linspace(block, last - block, spread).tolist()]
        starts = sorted({0, last, *mid})
    return [(r0, min(n, r0 + block)) for r0 in starts]


# ================================================================================================ key-code selectors (head-dim-128 kernels)
# Q_i and K_j are CODE_C * (sum of the unit vectors of a code): a pair of head dimensions, or a triple where a launch needs more codes
# than pairs give. A key of the query's code scores k C^2 (k = 2 or 3 dimensions); any other code shares at most k - 1 dimensions. A decoy
# is a key of the query's code at DECOY_MAG x the magnitude that the correct mask hides from that query: it would score k * 1.25 C^2 and win.
# 1.25, not 2: a decoy is an ordinary key to the queries that do see it, and at 2x a shared dimension (k - 1) * 2 C^2 would tie their target.
# Every gap is >= C^2 / 2 = 2048 in the score, 261 after the language model's 1/sqrt(128) log2(e), 330 after the vision heads'
# 1/sqrt(80) log2(e): the runner-up's exp2 is +0 in fp32, every score is an integer below 2^14 (exact in bf16 products and fp32 sums), and
# V on a grid of 1/16 in [-4, 4] keeps every sum of values exact. The output is then the mean of V over the visible keys of the query's code
# with the largest magnitude, bit for bit: bf16(fp32 sum * fp32(1 / count)).
CODE_C = 64.0
DECOY_MAG = 1.25
SLOT_MAX = 8                # keys per (KV head, code) at most


def code_table(n_needed, hd):
    """[n, k] head dimensions of every code: pairs of the first hd dimensions when there are enough of them, else triples."""
    k = 2 if hd * (hd - 1) // 2 >= n_needed else 3
    t = torch.combinations(torch.arange(hd), k)
    assert t.shape[0] >= n_needed, (hd, n_needed)
    return t


def int_v(shape, gen, device=None):
    """V on a coarse dyadic grid (integers in [-64, 64] / 16): every sum of values is exact in fp32 in any order."""
    return (torch.randint(-64, 65, shape, generator=gen, device=device).float() / 16)


def mean_bf16(sum_v, count):
    """bf16(fp32(sum) * fp32(1 / count)): the prefill kernel's O * (1 / l) with l the exact count of its P = 1 keys (IEEE division)."""
    inv = torch.ones_like(sum_v[..., :1], dtype=torch.float32) / count.float()[..., None]
    return (sum_v.float() * inv).bfloat16()


class Layout:
    """Which key rows each query row of a packed buffer sees. groups: row counts of the sequences (windows, frames) in buffer order;
    stride S: fixed-stride mode (group b at rows [b S, b S + len), the rest of its S rows padding). causal: a query sees its group's keys
    at positions <= its own. prefix_of[b]: a group whose rows sequence b also sees in full (kv_prefix), or -1."""

    def __init__(self, groups, causal, S=None, prefix_of=None, device="cpu"):
        self.groups, self.causal, self.S = list(groups), causal, S
        n = len(self.groups)
        lens = torch.tensor(self.groups, dtype=torch.long)
        if S is None:
            start = torch.cat([torch.zeros(1, dtype=torch.long), lens.cumsum(0)[:-1]])
            self.rows = int(lens.sum())
        else:
            assert all(x <= S for x in self.groups)
            start = torch.arange(n, dtype=torch.long) * S
            self.rows = n * S
        self.start, self.lens = start.to(device), lens.to(device)
        seq = torch.full((self.rows,), -1, dtype=torch.long)
        pos = torch.zeros(self.rows, dtype=torch.long)
        for b in range(n):
            a = int(start[b])
            seq[a:a + self.groups[b]] = b
            pos[a:a + (S or self.groups[b])] = torch.arange(S or self.groups[b])
        self.seq, self.pos = seq.to(device), pos.to(device)           # padding rows: seq -1 (no query, no key)
        self.prefix_of = torch.tensor(prefix_of if prefix_of is not None else [-1] * n, dtype=torch.long, device=device)
        self.device = device

    def visible(self, qr, kr):
        """Broadcast qr, kr (row indices; kr may hold -1 for none): does query row qr see key row kr?"""
        ok = kr >= 0
        kr = kr.clamp_min(0)
        qs, ks = self.seq[qr], self.seq[kr]
        own = (ks == qs) & (qs >= 0)
        if self.causal:
            own = own & (self.pos[kr] <= self.pos[qr])
        pre = (qs >= 0) & (ks >= 0) & (ks == self.prefix_of[qs.clamp_min(0)])
        return ok & (own | pre)

    def dense_visible(self):
        r = torch.arange(self.rows, device=self.device)
        return self.visible(r[:, None], r[None, :])

    def sample_visible_key(self, qr, gen, diag_frac=0.0):
        """A uniformly random visible key row for each query row qr (valid rows only); causal rows pick their own diagonal with
        probability diag_frac."""
        qs = self.seq[qr]
        own_n = (self.pos[qr] + 1) if self.causal else self.lens[qs]
        p = self.prefix_of[qs]
        pre_n = torch.where(p >= 0, self.lens[p.clamp_min(0)], 0)
        u = (torch.rand(qr.shape, generator=gen, device=self.device) * (pre_n + own_n)).long().clamp_max(pre_n + own_n - 1)
        if self.causal and diag_frac > 0:
            u = torch.where(torch.rand(qr.shape, generator=gen, device=self.device) < diag_frac, pre_n + own_n - 1, u)
        return torch.where(u < pre_n, self.start[p.clamp_min(0)] + u, self.start[qs] + u - pre_n)


class Selector:
    """A key-code selector fixture on a Layout: Hq query heads over Hkv KV heads (q head h reads KV head h // (Hq / Hkv)), codes over the
    first hd dimensions of 128-wide heads. Builds, in order: distinct codes for every key row of a KV head; tie groups (2 to 4 rows of one
    group share a code); decoys (a key near a query that the mask hides from it takes the code of that query's target, at DECOY_MAG); then
    every query's target, a visible key whose code the query takes. expected() is the closed form, brute() plain fp64 softmax attention."""

    def __init__(self, layout, Hq, Hkv, hd, gen, ties=0, decoy_frac=0.25, tie_sizes=(2, 3, 4), diag_frac=0.125, near=160):
        L, dev = layout, layout.device
        self.L, self.Hq, self.Hkv, self.hd, self.G = L, Hq, Hkv, hd, Hq // Hkv
        R = L.rows
        self.codes = code_table(R, hd).to(dev)
        n_codes = self.codes.shape[0]
        kc = torch.stack([torch.randperm(n_codes, generator=gen, device=dev)[:R] for _ in range(Hkv)], 1)       # [R, Hkv]
        mag = torch.ones(R, Hkv, device=dev)
        valid_rows = (L.seq >= 0).nonzero().squeeze(1)
        # tie groups: `ties` per KV head, members anywhere in one group (distant key tiles in a long sequence)
        for g in range(Hkv):
            for t in range(ties):
                b = int(L.seq[valid_rows[int(torch.randint(len(valid_rows), (1,), generator=gen, device=dev))]])
                n = L.groups[b]
                size = min(n, tie_sizes[t % len(tie_sizes)])
                if size < 2:
                    continue
                rows = L.start[b] + torch.randperm(n, generator=gen, device=dev)[:size]
                kc[rows, g] = int(kc[rows[0], g])
        # decoys: a query row, one of its heads, and a key row within `near` rows (or just past its prefix) that it must not see
        q_rows = torch.arange(R, device=dev)
        is_decoy = torch.zeros(R, Hkv, dtype=torch.bool, device=dev)
        self.victims = []
        n_vic = int(decoy_frac * len(valid_rows))
        if n_vic > 0:
            vq = valid_rows[torch.randint(len(valid_rows), (n_vic,), generator=gen, device=dev)]
            vh = torch.randint(Hq, (n_vic,), generator=gen, device=dev)
            delta = torch.randint(-near, near + 1, (n_vic,), generator=gen, device=dev)
            dk = vq + delta
            p = L.prefix_of[L.seq[vq]]
            past_prefix = L.start[p.clamp_min(0)] + L.lens[p.clamp_min(0)] + delta.abs() % 130
            dk = torch.where((p >= 0) & (torch.rand(n_vic, generator=gen, device=dev) < 0.5), past_prefix, dk)
            ok = (dk >= 0) & (dk < R)
            vq, vh, dk = vq[ok], vh[ok], dk[ok]
            ok = ~L.visible(vq, dk)
            vq, vh, dk = vq[ok], vh[ok], dk[ok]
            g = vh // self.G
            key = dk * Hkv + g                                   # one victim per (key row, KV head)
            uniq, inv = torch.unique(key, return_inverse=True)
            first = torch.full((len(uniq),), len(key), device=dev, dtype=torch.long).scatter_reduce(0, inv, torch.arange(len(key), device=dev), "amin")
            vq, vh, dk, g = vq[first], vh[first], dk[first], g[first]
            is_decoy[dk, g] = True
            tgt = L.sample_visible_key(vq, gen)
            ok = ~is_decoy[tgt, g]
            is_decoy[dk[~ok], g[~ok]] = False
            vq, vh, dk, g, tgt = vq[ok], vh[ok], dk[ok], g[ok], tgt[ok]
            kc[dk, g] = kc[tgt, g]
            mag[dk, g] = DECOY_MAG
            self.victims = (vq, vh, dk, tgt)
        # every query's target, then its code
        target = torch.zeros(R, Hq, dtype=torch.long, device=dev)
        for h in range(Hq):
            target[valid_rows, h] = L.sample_visible_key(valid_rows, gen, diag_frac)
        if len(self.victims):
            vq, vh, dk, tgt = self.victims
            target[vq, vh] = tgt
        self.key_code, self.mag = kc, mag
        qc = kc[target, (torch.arange(Hq, device=dev) // self.G)[None, :]]                      # [R, Hq]
        qc[L.seq < 0] = torch.randint(n_codes, (int((L.seq < 0).sum()), Hq), generator=gen, device=dev)
        self.q_code = qc
        self.v = int_v((R, Hkv, hd), gen, dev)

    def unit_rows(self, code, scale):
        """[..., 128] rows scale * (sum of the code's unit vectors)."""
        x = torch.zeros(*code.shape, 128, device=code.device)
        d = self.codes[code]
        x.scatter_(-1, d, scale[..., None].expand(*code.shape, d.shape[-1]) if torch.is_tensor(scale) else torch.full(d.shape, scale, device=code.device))
        return x

    def tensors(self):
        """q [R, Hq, 128], k / v [R, Hkv, 128] as fp32 (exact in bf16); V columns past hd are 0."""
        q = self.unit_rows(self.q_code, CODE_C)
        k = self.unit_rows(self.key_code, CODE_C * self.mag)
        v = torch.zeros(self.L.rows, self.Hkv, 128, device=self.L.device)
        v[..., :self.hd] = self.v
        return q, k, v

    def expected(self, heads=None):
        """Closed form [R, Hq, hd] bf16 (padding query rows +0) and the winner count [R, Hq] (0 for padding rows)."""
        L, dev, R, Hkv = self.L, self.L.device, self.L.rows, self.Hkv
        keyed = (L.seq >= 0).nonzero().squeeze(1)
        n_codes = self.codes.shape[0]
        slot = (torch.arange(Hkv, device=dev)[None, :] * n_codes + self.key_code[keyed]).reshape(-1)     # [n_keyed * Hkv]
        krow = keyed[:, None].expand(-1, Hkv).reshape(-1)
        order = torch.argsort(slot, stable=True)
        slot, krow = slot[order], krow[order]
        uniq, counts = torch.unique_consecutive(slot, return_counts=True)
        assert int(counts.max()) <= SLOT_MAX, int(counts.max())
        first = torch.cumsum(counts, 0) - counts
        rank = torch.arange(len(slot), device=dev) - torch.repeat_interleave(first, counts)
        members = torch.full((len(uniq), SLOT_MAX), -1, dtype=torch.long, device=dev)
        members[torch.repeat_interleave(torch.arange(len(uniq), device=dev), counts), rank] = krow
        out = torch.zeros(R, self.Hq, self.hd, dtype=torch.bfloat16, device=dev)
        cnt = torch.zeros(R, self.Hq, dtype=torch.long, device=dev)
        rows = (L.seq >= 0).nonzero().squeeze(1)
        for h in (range(self.Hq) if heads is None else heads):
            g = h // self.G
            qslot = g * n_codes + self.q_code[rows, h]
            idx = torch.searchsorted(uniq, qslot)
            assert bool((uniq[idx.clamp_max(len(uniq) - 1)] == qslot).all())
            m = members[idx]                                                        # [n, SLOT_MAX]
            vis = L.visible(rows[:, None], m)
            mg = torch.where(vis, self.mag[m.clamp_min(0), g], 0.0)
            win = vis & (mg == mg.amax(-1, keepdim=True))
            c = win.sum(-1)
            assert bool((c >= 1).all())
            s = (self.v[m.clamp_min(0), g].double() * win[..., None]).sum(1)
            out[rows, h] = mean_bf16(s, c)
            cnt[rows, h] = c
        return out, cnt

    def brute(self, scale, visible=None, heads=None):
        """Plain fp64 softmax attention over every key row with `visible` [R, R] (default the layout's mask): [R, Hq, hd] (rows with no
        visible key: 0), and the exp2-domain gap between each row's best score and the best one below it (tied winners share the best)."""
        q, k, v = (t.double() for t in self.tensors())
        vis = self.L.dense_visible() if visible is None else visible
        outs, gaps = [], []
        for h in (range(self.Hq) if heads is None else heads):
            g = h // self.G
            s = (q[:, h] @ k[:, g].t()).masked_fill(~vis, float("-inf"))
            top = s.amax(-1, keepdim=True)
            gaps.append((top - s.masked_fill(s == top, float("-inf")).amax(-1, keepdim=True)).squeeze(-1) * scale / LN2)
            p = torch.softmax(s, -1).nan_to_num(0.0)
            outs.append(p @ v[:, g, :self.hd])
        return torch.stack(outs, 1), torch.stack(gaps, 1)


def decode_selector(lens, Hq, Hkv, cap, chunk, gen, device="cpu"):
    """Key-code selectors over a K/V cache [B, Hkv, cap, 128] for the flash-decoding kernel, keys of split s at slots [s chunk, (s + 1)
    chunk). Distinct pair codes per (sequence, KV head); q head h of sequence b puts its code on the slots of one placement: the first key,
    the last live key, the last key of split 0 (a split that ends exactly at len when len = chunk), a 2-tie across the first split
    boundary, a 4-tie across the first two, a 2-tie across the boundary into the last split. Placements of heads of one KV head may merge
    ties; each query takes its first slot's final code. Slots at or past len hold NaN. Returns (q [B, Hq, 128], kc, vc as fp32,
    expected bf16 [B, Hq, 128] = bf16(fp32 sum / count) as the merge divides, count [B, Hq])."""
    B, G = len(lens), Hq // Hkv
    codes = code_table(cap, 128).to(device)
    kcode = torch.stack([torch.randperm(codes.shape[0], generator=gen, device=device)[:cap] for _ in range(B * Hkv)]).view(B, Hkv, cap)
    first = torch.zeros(B, Hq, dtype=torch.long)
    for b, n in enumerate(lens):
        last = (n - 1) // chunk * chunk
        for h in range(Hq):
            pos = [[0], [n - 1], [min(chunk, n) - 1], [chunk - 1, chunk], [chunk - 1, chunk, 2 * chunk - 1, 2 * chunk],
                   [last - 1, last]][(b + 3 * h) % 6]
            pos = sorted({p for p in pos if 0 <= p < n}) or [n - 1]
            kcode[b, h // G, pos[1:]] = int(kcode[b, h // G, pos[0]])
            first[b, h] = pos[0]
    bi = torch.arange(B)[:, None]
    qcode = kcode[bi, torch.arange(Hq)[None, :] // G, first]                                   # [B, Hq]
    q = torch.zeros(B, Hq, 128, device=device).scatter_(-1, codes[qcode], CODE_C)
    k = torch.zeros(B, Hkv, cap, 128, device=device).scatter_(-1, codes[kcode], CODE_C)
    v = int_v((B, Hkv, cap, 128), gen, device)
    live = torch.arange(cap, device=device)[None, :] < torch.tensor(lens, device=device)[:, None]           # [B, cap]
    win = (kcode[:, torch.arange(Hq) // G] == qcode[..., None]) & live[:, None, :]                           # [B, Hq, cap]
    s = torch.einsum("bhc,bhcd->bhd", win.double(), v[:, torch.arange(Hq) // G].double())
    cnt = win.sum(-1)
    want = (s.float() / cnt.float()[..., None]).bfloat16()
    k[~live[:, None, :, None].expand_as(k)] = float("nan")
    v[~live[:, None, :, None].expand_as(v)] = float("nan")
    return q, k, v, want, cnt
