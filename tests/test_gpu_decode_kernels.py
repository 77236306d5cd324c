"""Kernel-level parity of the greedy decode loops on a real H100, through the C ABI (vqa_op_*): the Qwen2.5-VL K/V cache write,
flash-decoding attention and greedy token selection, and the CLIP-FlanT5 decoder self-attention (scoring kernel and cached kernel).

References are plain torch in fp64 built from the same bf16 inputs, rounded where the kernel (and the HF module it mirrors) rounds.
Cache slots at or past a sequence's live length hold a bf16 NaN, so any read of one shows in the output, and caches / outputs sit between
sentinel guard bands that must come back bit-identical, so an out-of-range write shows too. Each group also checks that its fixture
discriminates: the reference with a plausible kernel mistake applied moves by several times the tolerance."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

SENTINEL = 0x7FA5          # a bf16 NaN bit pattern, distinct from the NaN any arithmetic produces (0x7FC0)
GUARD = 256                # guard-band elements on either side (512 bytes: keeps 16-byte alignment)


@pytest.fixture(scope="module")
def ops():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    from t2v_metrics_b200.engine import ops as _ops
    return _ops


class Guarded:
    """A bf16 tensor of `shape` inside a sentinel-filled buffer with GUARD elements before and after; the tensor starts as sentinel."""

    def __init__(self, shape):
        self.n = math.prod(shape)
        self.raw = torch.full((GUARD + self.n + GUARD,), SENTINEL, dtype=torch.int16, device="cuda")
        self.t = self.raw[GUARD:GUARD + self.n].view(torch.bfloat16).view(shape)

    def bits(self):
        return self.t.view(torch.int16)

    def guards_intact(self):
        return bool((self.raw[:GUARD] == SENTINEL).all()) and bool((self.raw[GUARD + self.n:] == SENTINEL).all())


def bf16_ulp(x):
    """Spacing of bf16 numbers at |x| (8 significant bits)."""
    return torch.exp2(torch.floor(torch.log2(x.abs().clamp_min(2.0 ** -100))) - 7)


# ================================================================================================ Qwen decode attention
QWEN_HEADS = [(28, 4), (16, 2), (40, 8), (64, 8), (1, 1), (2, 1), (4, 1)]     # 7B, 3B, 32B, 72B; G = 7, 8, 5, 8, 1, 2, 4
SCALE = 1.0 / math.sqrt(128.0)
Q0 = 8.0                   # dimension 0 of every query: a key's dimension 0 sets its score offset for every head of its group


def sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


def split_rule(B, Hkv, cap):
    """The generation plan's split count (decode_attn_splits): two CTAs per SM, at least 16 keys per split."""
    return max(1, min((2 * sm_count() + B * Hkv - 1) // (B * Hkv), (cap + 15) // 16))


def ragged_lengths(cap, chunk):
    cand = [1, 3, chunk - 1, chunk, chunk + 1, chunk // 2 + 1, 2 * chunk + 3, cap - chunk - 1, cap - 1, cap]
    return sorted(set(x for x in cand if 1 <= x <= cap))


def build_decode_case(Hq, Hkv, cap, lens, plants, chunk, seed):
    """Packed query rows, NaN-poisoned caches and the live lengths. Keys carry a score offset per production split (+50 / -50 / 0, so split
    maxima sit 100 apart) on top of unit noise; in some rows one key is planted ~20 above the row's maximum at a boundary position:
    plant 1 at key 0, 2 at key len - 1, 3 at the first key of the last non-empty split, 4 at the last key of split 0."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    B, G = len(lens), Hq // Hkv
    ld = (Hq + 2 * Hkv) * 128
    q = torch.randn(B, Hq, 128, device="cuda", generator=g)
    q[..., 0] = Q0
    k = torch.randn(B, Hkv, cap, 128, device="cuda", generator=g)
    v = torch.randn(B, Hkv, cap, 128, device="cuda", generator=g)
    split = torch.arange(cap, device="cuda") // chunk
    offset = torch.tensor([50.0, -50.0, 0.0], device="cuda")[split % 3]
    unit = Q0 * SCALE                      # score per unit of key dimension 0
    k[..., 0] = offset / unit
    planted = []
    for b, (L, kind) in enumerate(zip(lens, plants)):
        last_split = (L - 1) // chunk
        pos = {1: 0, 2: L - 1, 3: last_split * chunk if last_split >= 1 else None, 4: chunk - 1 if chunk - 1 < L - 1 else None}.get(kind)
        if pos is not None:
            top = float(offset[:L].max())
            k[b, :, pos, 0] = (top + 20.0) / unit
            planted.append((b, pos))
    qkv = torch.full((B, ld), float("nan"), device="cuda")          # the row's K / V columns are never read by the attention
    qkv[:, :Hq * 128] = q.reshape(B, Hq * 128)
    qkv = qkv.bfloat16()
    kc, vc = k.bfloat16(), v.bfloat16()
    live = torch.arange(cap, device="cuda")[None, :] < torch.tensor(lens, device="cuda")[:, None]
    kc[~live[:, None, :, None].expand_as(kc)] = float("nan")
    vc[~live[:, None, :, None].expand_as(vc)] = float("nan")
    lens_t = torch.tensor(lens, dtype=torch.int32, device="cuda")
    gen_len = torch.tensor([1 + (7 * b) % L for b, L in enumerate(lens)], dtype=torch.int32, device="cuda")   # 1 <= gen_len <= len
    seq_lens = lens_t - gen_len
    return qkv, kc, vc, seq_lens, gen_len, lens_t, planted


def ref_decode_attention(qkv, kc, vc, lens, Hq, drop=None, merge_chunk=None):
    """fp64 attention of each query row over its live keys. drop [B, cap] bool: keys removed. merge_chunk: the merge of the per-split
    partials with every split weighted 1 instead of e^(m_s - M) (the merge without its rescale)."""
    B, Hkv, cap, _ = kc.shape
    G = Hq // Hkv
    q = qkv[:, :Hq * 128].double().view(B, Hkv, G, 128) * SCALE
    valid = torch.arange(cap, device="cuda")[None, :] < lens[:, None].long()
    if drop is not None:
        valid = valid & ~drop
    k = torch.where(valid[:, None, :, None], kc.double(), 0.0)
    v = torch.where(valid[:, None, :, None], vc.double(), 0.0)
    s = (q @ k.transpose(-1, -2)).masked_fill(~valid[:, None, None, :], float("-inf"))       # [B, Hkv, G, cap]
    if merge_chunk is None:
        out = torch.softmax(s, -1) @ v
    else:
        n = -(-cap // merge_chunk)
        pad = n * merge_chunk - cap
        s4 = torch.nn.functional.pad(s, (0, pad), value=float("-inf")).view(B, Hkv, G, n, merge_chunk)
        v4 = torch.nn.functional.pad(v, (0, 0, 0, pad)).view(B, Hkv, n, merge_chunk, 128)
        m = s4.amax(-1, keepdim=True)
        e = torch.where(m > float("-inf"), torch.exp(s4 - m), 0.0)
        out = torch.einsum("bhgsc,bhscd->bhgd", e, v4) / e.sum((-1, -2))[..., None]
    return out.reshape(B, Hq * 128)


def decode_tolerance(ref, vc_live_max):
    return 2.0 ** -8 * ref.abs() + 2.0 ** -10 * vc_live_max


def run_decode_attention(ops, qkv, kc, vc, seq_lens, gen_len, Hq, splits):
    """The op with a guarded output (row stride Hq * 128 + 64, one sentinel row before and after); returns (out, splits used)."""
    B = qkv.shape[0]
    ldo = Hq * 128 + 64
    buf = torch.full(((B + 2) * ldo,), SENTINEL, dtype=torch.int16, device="cuda")
    out = buf.view(torch.bfloat16).view(B + 2, ldo)[1:B + 1, :Hq * 128]
    _, used = ops.decode_attention(qkv, kc, vc, seq_lens, gen_len, Hq, SCALE, splits=splits, out=out)
    torch.cuda.synchronize()
    written = torch.zeros(B + 2, ldo, dtype=torch.bool, device="cuda")
    written[1:B + 1, :Hq * 128] = True
    assert bool((buf.view(B + 2, ldo)[~written] == SENTINEL).all()), "decode attention wrote outside its output rows"
    return out.float(), used


def check_decode_attention(ops, Hq, Hkv, cap, lens, plants, seed, discriminate):
    B = len(lens)
    rule = split_rule(B, Hkv, cap)
    chunk = -(-cap // rule)
    qkv, kc, vc, seq_lens, gen_len, lens_t, planted = build_decode_case(Hq, Hkv, cap, lens, plants, chunk, seed)
    ref = ref_decode_attention(qkv, kc, vc, lens_t, Hq)
    vmax = float(vc.float().nan_to_num(0.0).abs().max())
    tol = decode_tolerance(ref, vmax)
    outs = {}
    for splits in sorted({1, 0, -(-cap // 16)}):
        out, used = run_decode_attention(ops, qkv, kc, vc, seq_lens, gen_len, Hq, splits)
        if splits == 0:
            assert used == rule, (used, rule)          # the op's default is the generation plan's rule
        assert bool(torch.isfinite(out).all()), (splits, "a poisoned slot was read")
        err = (out - ref).abs()
        bad = err > tol
        assert not bool(bad.any()), (used, int(bad.sum()), float(err.max()), float((err / tol).max()))
        outs[used] = out
    first = next(iter(outs.values()))
    for used, out in outs.items():       # split counts only reorder fp32 sums: at most one bf16 ulp apart
        assert bool(((out - first).abs() <= bf16_ulp(torch.maximum(out.abs(), first.abs()).clamp_min(2.0 ** -6))).all()), used
    if discriminate:
        # the data must catch a subtly wrong kernel: each mistake moves some output by more than 8x the tolerance
        idx = torch.arange(cap, device="cuda")
        mistakes = {
            "drops key len - 1": ref_decode_attention(qkv, kc, vc, lens_t, Hq, drop=idx[None, :] == (lens_t.long() - 1)[:, None]),
            "drops each split's first key": ref_decode_attention(qkv, kc, vc, lens_t, Hq, drop=(idx % chunk == 0)[None, :].expand(B, cap)),
            "merges without the rescale": ref_decode_attention(qkv, kc, vc, lens_t, Hq, merge_chunk=chunk),
        }
        for what, wrong in mistakes.items():
            moved = ((wrong - ref).abs() / tol).nan_to_num(0.0)
            assert float(moved.max()) > 8.0, (what, float(moved.max()))
    return planted


@pytest.mark.parametrize("cap", [17, 320 + 128])
@pytest.mark.parametrize("Hq,Hkv", QWEN_HEADS)
def test_decode_attention_every_group_size(ops, Hq, Hkv, cap):
    """Every group size the dispatch instantiates, at the family's head counts. cap 17 makes two splits with keys in the last partial one;
    448 is the benchmark's prompt + generation capacity. Ragged lengths around the production chunk (1, chunk - 1, chunk, chunk + 1,
    lengths that leave trailing splits empty, cap), each twice with different planted keys; splits 1, the rule's and ceil(cap / 16)."""
    B = 20
    chunk = -(-cap // split_rule(B, Hkv, cap))
    L = ragged_lengths(cap, chunk)
    lens = [L[i % len(L)] for i in range(B)]
    plants = [(i + i // len(L)) % 5 for i in range(B)]       # a length's repeats carry different planted keys
    planted = check_decode_attention(ops, Hq, Hkv, cap, lens, plants, seed=Hq * 1000 + cap, discriminate=True)
    assert len(planted) >= 4


@pytest.mark.parametrize("B,cap", [(1, 32768), (128, 4096)])
@pytest.mark.parametrize("Hq,Hkv", [(28, 4), (16, 2)])
def test_decode_attention_long_and_wide_caches(ops, Hq, Hkv, B, cap):
    """B = 1 over a 32k-slot cache (the rule's 66 splits of 497 keys at 7B: odd-sized chunks) and B = 128 over 4096 slots (one split of
    every key). B = 1 runs a full cache and one whose live keys end just past a split edge."""
    torch.manual_seed(B + cap)
    chunk = -(-cap // split_rule(B, Hkv, cap))
    if B == 1:
        check_decode_attention(ops, Hq, Hkv, cap, [cap], [2], seed=1, discriminate=False)
        check_decode_attention(ops, Hq, Hkv, cap, [3 * chunk + 1], [3], seed=2, discriminate=False)
    else:
        lens = ragged_lengths(cap, chunk)
        lens = lens + torch.randint(1, cap + 1, (B - len(lens),)).tolist()
        check_decode_attention(ops, Hq, Hkv, cap, lens, [i % 5 for i in range(B)], seed=3, discriminate=False)


# ================================================================================================ Qwen K/V cache write
@pytest.mark.parametrize("Hq,Hkv", [(28, 4), (64, 8)])
def test_kv_cache_write_prefill_and_decode(ops, Hq, Hkv):
    """Bit-exact against torch indexing. Prefill: ragged seq_lens in padded rows (padded rows must not be written: their slots keep the
    sentinel). Decode: one row per sequence at seq_lens + gen_len - 1, including seq_lens = S with gen_len = max_new (slot cap - 1)."""
    torch.manual_seed(Hq)
    B, S, max_new = 6, 37, 6
    cap = S + max_new
    ld, k0, v0 = (Hq + 2 * Hkv) * 128, Hq * 128, (Hq + Hkv) * 128
    seq_lens = [S, 1, 20, S - 1, 9, S]
    sl = torch.tensor(seq_lens, dtype=torch.int32, device="cuda")
    qkv = torch.randn(B * S, ld, device="cuda").bfloat16()
    kc, vc = Guarded((B, Hkv, cap, 128)), Guarded((B, Hkv, cap, 128))
    ops.kv_cache_write(qkv, k0, v0, Hkv, S, sl, kc.t, vc.t)
    exp_k = torch.full((B, Hkv, cap, 128), SENTINEL, dtype=torch.int16, device="cuda")
    exp_v = exp_k.clone()
    rows = qkv.view(B, S, ld).view(torch.int16)
    for b, L in enumerate(seq_lens):
        exp_k[b, :, :L] = rows[b, :L, k0:k0 + Hkv * 128].reshape(L, Hkv, 128).transpose(0, 1)
        exp_v[b, :, :L] = rows[b, :L, v0:v0 + Hkv * 128].reshape(L, Hkv, 128).transpose(0, 1)
    torch.cuda.synchronize()
    assert torch.equal(kc.bits(), exp_k) and torch.equal(vc.bits(), exp_v)
    assert kc.guards_intact() and vc.guards_intact()
    # decode: one new row per sequence
    gen_len = [max_new, 1, 3, 2, 6, 4]
    gl = torch.tensor(gen_len, dtype=torch.int32, device="cuda")
    step = torch.randn(B, ld, device="cuda").bfloat16()
    ops.kv_cache_write(step, k0, v0, Hkv, 1, sl, kc.t, vc.t, gen_len=gl)
    srow = step.view(torch.int16)
    for b in range(B):
        slot = seq_lens[b] + gen_len[b] - 1
        exp_k[b, :, slot] = srow[b, k0:k0 + Hkv * 128].view(Hkv, 128)
        exp_v[b, :, slot] = srow[b, v0:v0 + Hkv * 128].view(Hkv, 128)
    assert seq_lens[0] + gen_len[0] - 1 == cap - 1
    torch.cuda.synchronize()
    assert torch.equal(kc.bits(), exp_k) and torch.equal(vc.bits(), exp_v)
    assert kc.guards_intact() and vc.guards_intact()


# ================================================================================================ greedy selection
def processed_scores(logits, bitmap, penalty):
    """HF's processing in fp32: bf16 logits -> fp32 -> RepetitionPenaltyLogitsProcessor on the bitmap's ids."""
    x = logits.float().cpu()
    if bitmap is None:
        return x
    V = x.shape[1]
    words = bitmap.cpu().long() & 0xFFFFFFFF
    ids = torch.arange(V)
    hit = ((words[:, ids // 32] >> (ids % 32)) & 1).bool()
    return torch.where(hit, torch.where(x < 0, x * penalty, x / penalty), x)


class SelectState:
    """The generation state greedy_select_kernel keeps on the device, and a Python model of one step."""

    def __init__(self, B, V, max_new, bitmap=None, first_pos=None, lengths=None, done=None):
        self.tokens = torch.full((B, max_new), -1, dtype=torch.int32)
        self.lengths = torch.zeros(B, dtype=torch.int32) if lengths is None else lengths.clone()
        self.done = torch.zeros(B, dtype=torch.int32) if done is None else done.clone()
        self.n_done = torch.tensor([int(self.done.sum())], dtype=torch.int32)
        self.all_done = torch.zeros(1, dtype=torch.int32)
        self.next_ids = torch.full((B,), -3, dtype=torch.int32)
        self.bitmap = bitmap.clone() if bitmap is not None else None
        self.first_pos = first_pos
        self.pos3 = torch.full((3, B), -7, dtype=torch.int32) if first_pos is not None else None
        self.B, self.V, self.max_new = B, V, max_new

    def fields(self):
        f = dict(tokens=self.tokens, lengths=self.lengths, done=self.done, n_done=self.n_done, all_done=self.all_done, next_ids=self.next_ids)
        if self.bitmap is not None:
            f["bitmap"] = self.bitmap
        if self.pos3 is not None:
            f["pos3"] = self.pos3
        return f

    def to_device(self):
        d = SelectState.__new__(SelectState)
        d.__dict__.update({k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in self.__dict__.items()})
        return d

    def step_ref(self, logits, eos_ids, penalty):
        best = processed_scores(logits, self.bitmap, penalty).argmax(-1)        # torch.argmax: the first maximum
        for b in range(self.B):
            if self.done[b]:
                continue
            tok, t = int(best[b]), int(self.lengths[b])
            self.tokens[b, t] = tok
            self.lengths[b] = t + 1
            if self.bitmap is not None:
                w = int(self.bitmap[b, tok // 32]) & 0xFFFFFFFF | (1 << (tok % 32))
                self.bitmap[b, tok // 32] = w - (1 << 32) if w >= 1 << 31 else w
            self.next_ids[b] = tok
            if self.pos3 is not None:
                self.pos3[:, b] = int(self.first_pos[b]) + t
            if t + 1 >= self.max_new or tok in eos_ids:
                self.done[b] = 1
                self.n_done[0] += 1
                if int(self.n_done[0]) == self.B:
                    self.all_done[0] = 1
        return best

    def step_kernel(self, ops, logits, eos, penalty):
        ops.greedy_select(logits, self.tokens, self.lengths, self.done, self.n_done, self.all_done, self.next_ids, eos_ids=eos,
                          pen_bitmap=self.bitmap, repetition_penalty=penalty, first_pos=self.first_pos, pos3=self.pos3)


def assert_same_state(dev, ref, what):
    for name, want in ref.fields().items():
        got = dev.fields()[name].cpu()
        assert torch.equal(got, want), (what, name, got, want)


def tie_rows(V, gen):
    """Rows that probe the selection rule, one expected winner each (under no penalty):
    0 random; 1 maxima repeated in the same warp, across warps and past id 1024; 2 maxima only past id 1024 and in later passes of
    lower threads; 3 -0.0 before +0.0 under negative values; 4 +0.0 before -0.0; 5 a constant row; 6 the maximum only at id V - 1;
    7 a row of negatives."""
    rows = torch.randn(8, V, generator=gen) * 2 - 1
    rows = rows.clamp(max=3.0)
    ids = lambda xs: sorted(set(i % V for i in xs))
    rows[1, ids([37, 35, 100, 1030, 5000, V - 1])] = 5.0
    rows[2, ids([2047, 1030, 1500, 5000, V - 1])] = 5.0
    rows[3] = -rows[3].abs() - 1.0
    rows[3, ids([3])] = -0.0
    rows[3, ids([900])] = 0.0
    rows[4] = -rows[4].abs() - 1.0
    rows[4, ids([3])] = 0.0
    rows[4, ids([900])] = -0.0
    rows[5] = 1.0
    rows[6, V - 1] = 4.0
    rows[7] = -rows[7].abs() - 0.5
    return rows.bfloat16()


@pytest.mark.parametrize("penalty", [1.0, 1.25])
@pytest.mark.parametrize("V", [152064, 32128, 1001, 5])
def test_greedy_select_ties_and_penalty(ops, V, penalty):
    """One step, bit-exact. V = 5 leaves most threads without an id; 1001 and 32128 end in a partial bitmap word (whose bits past V are
    set and must be ignored). With the penalty: random prompt bits, plus a tie the penalty creates (bf16 2.5 / 1.25 = 2.0 against an
    unpenalised 2.0) in either id order. Rows that are finished, at their last token, or whose token is an EOS id cover the bookkeeping."""
    gen = torch.Generator().manual_seed(V)
    logits = tie_rows(V, gen)
    B = logits.shape[0]
    bitmap = None
    if penalty != 1.0:
        words = -(-V // 32)
        bits = (torch.rand(B, words * 32, generator=gen) < 0.3)
        bits[:, V:] = True
        if V > 60:
            for b, (a, c) in ((0, (10, 50)), (6, (50, 10))):      # id a: 2.5 penalised to 2.0; id c: an unpenalised 2.0
                logits[b] = logits[b].clamp(max=1.5)
                logits[b, a], logits[b, c] = 2.5, 2.0
                bits[b, a], bits[b, c] = True, False
            logits[6, V - 1] = 1.0
        packed = (bits.view(B, words, 32).long() << torch.arange(32)).sum(-1)
        bitmap = torch.where(packed >= 1 << 31, packed - (1 << 32), packed).to(torch.int32)
    max_new = 4
    lengths = torch.tensor([0, 1, 2, 3, 0, 1, 2, 0], dtype=torch.int32)      # row 3 reaches max_new
    done = torch.tensor([0, 0, 0, 0, 0, 0, 0, 1], dtype=torch.int32)         # row 7 finished earlier: untouched
    first_pos = torch.arange(B, dtype=torch.int32) * 11 + 40
    ref = SelectState(B, V, max_new, bitmap, first_pos, lengths, done)
    best = ref.step_ref(logits, [], penalty)
    eos = [int(best[5])]                                  # row 5's token is an EOS id this time: it finishes at its second token
    ref = SelectState(B, V, max_new, bitmap, first_pos, lengths, done)
    ref.step_ref(logits, eos, penalty)
    dev = SelectState(B, V, max_new, bitmap, first_pos, lengths, done).to_device()
    dev.first_pos = first_pos.cuda()
    dev.step_kernel(ops, logits.cuda(), torch.tensor(eos, dtype=torch.int32, device="cuda"), penalty)
    torch.cuda.synchronize()
    assert_same_state(dev, ref, (V, penalty))
    # the fixture does rest on the rule: ties to the highest id, or a skipped penalty, would pick other tokens
    if V >= 5001 and penalty == 1.0:
        last = V - 1 - processed_scores(logits, None, 1.0).flip(-1).argmax(-1)
        assert int(last[1]) != int(best[1]) and int(last[2]) != int(best[2])
    if V > 60 and penalty != 1.0:
        assert int(best[0]) == 10 and int(best[6]) == 10                  # the penalty's tie, both id orders
        assert int(logits[6].float().argmax()) == 50                      # unpenalised, the other id wins


@pytest.mark.parametrize("style", ["qwen", "t5"])
def test_greedy_select_decode_loop_state_machine(ops, style):
    """40 steps at B = 7 with fresh, tie-rich logits every step against a Python state machine, comparing the whole state after every step:
    tokens (-1 past the end), lengths, penalty bits (the EOS token's included), next ids, positions on all three axes, done, n_done and
    all_done, which must rise exactly on the step the last rows finish -- here two at once, one by EOS and one by length. Rows finish at
    scheduled steps by EOS (two of them together) and stay untouched afterwards. The T5 loop passes no penalty and no positions."""
    B, V, max_new = 7, 1001, 40
    eos_ids = [2, 999]
    finish = {6: 0, 0: 5, 1: 12, 2: 12, 5: 20, 4: 39}        # row -> step of its EOS; row 3 runs to max_new, ending at step 39 as well
    gen = torch.Generator().manual_seed(4)
    penalty, bitmap, first_pos = 1.0, None, None
    if style == "qwen":
        penalty = 1.25
        words = -(-V // 32)
        bits = torch.rand(B, words * 32, generator=gen) < 0.2
        packed = (bits.view(B, words, 32).long() << torch.arange(32)).sum(-1)
        bitmap = torch.where(packed >= 1 << 31, packed - (1 << 32), packed).to(torch.int32)
        first_pos = torch.randint(5, 900, (B,), generator=gen, dtype=torch.int32)
    ref = SelectState(B, V, max_new, bitmap, first_pos)
    dev = ref.to_device()
    eos_dev = torch.tensor(eos_ids, dtype=torch.int32, device="cuda")
    for t in range(max_new):
        logits = (torch.randint(-6, 7, (B, V), generator=gen).float() / 2)
        logits[:, eos_ids] = -20.0
        for b, step in finish.items():
            if step == t:
                logits[b, eos_ids[b % 2]] = 50.0
        logits = logits.bfloat16()
        before = ref.done.clone()
        ref.step_ref(logits, eos_ids, penalty)
        dev.step_kernel(ops, logits.cuda(), eos_dev, penalty)
        torch.cuda.synchronize()
        assert_same_state(dev, ref, t)
        assert int(ref.all_done[0]) == (1 if t == max_new - 1 else 0), t
        assert int(ref.n_done[0]) == sum(1 for s in list(finish.values()) + [max_new - 1] if s <= t)
        newly = (ref.done - before).nonzero().flatten().tolist()
        assert newly == sorted([b for b, s in finish.items() if s == t] + ([3] if t == max_new - 1 else []))
    assert bool((ref.tokens[6, 1:] == -1).all()) and int(ref.lengths[6]) == 1


# ================================================================================================ T5 decoder self-attention
NB, MD = 32, 128           # relative_attention_num_buckets, relative_attention_max_distance


def t5_data(shape, gen):
    """Values on a 1/4 grid in [-0.5, 0.5]: every q.k is a multiple of 1/16 below 16 in magnitude, exact in fp32 whatever the summation
    order, so the kernel's score and the reference's round to the same bf16."""
    return (torch.randint(-2, 3, shape, generator=gen, device="cuda").float() / 4).bfloat16()


def t5_rel_emb(H, gen):
    """A distinct value per bucket (and head), 0.75 apart across [-12, 11.25]: a bucket off by one moves the score by >= 0.75."""
    perm = torch.stack([torch.randperm(NB, generator=gen, device="cuda") for _ in range(H)], 1)
    return (perm.float() * 0.75 - 12.0).bfloat16()


def t5_lut(ops, bidirectional=False):
    return ops.t5_bucket_lut(bidirectional, NB, MD).cuda()


def ref_t5_row(q, k, v, tq, rel_emb, round_scores, buckets=None):
    """fp64 decoder self-attention of one query at position tq over keys 0..tq (q [H, 64], k / v [tq + 1, H, 64]) -> [H, 64]:
    unscaled scores, bf16-rounded before and after the bias add when round_scores, softmax, P rounded to bf16 before P.V."""
    from oracle import clipt5_oracle as orc
    rel = torch.arange(tq + 1, device="cuda") - tq
    bucket = orc.relative_position_bucket(rel, False, NB, MD) if buckets is None else buckets(rel)
    s = torch.einsum("hd,khd->hk", q.double(), k.double())
    if round_scores:
        s = s.bfloat16().double()
    s = s + rel_emb.double()[bucket].t()
    if round_scores:
        s = s.bfloat16().double()
    p = torch.softmax(s, -1).bfloat16().double()
    return torch.einsum("hk,khd->hd", p, v.double())


def t5_tolerance(ref, vmax):
    # bf16 output rounding plus P-rounding flips (each at most one bf16 ulp of its weight): sum_k ulp(p_k) |v_k| <= 2^-8 max|V|
    return 2.0 ** -8 * ref.abs() + 1.25 * 2.0 ** -8 * vmax


def t5_mistakes():
    from oracle import clipt5_oracle as orc
    return {
        "bucket shifted by one": lambda rel: (orc.relative_position_bucket(rel, False, NB, MD) + 1).clamp(max=NB - 1),
        "bidirectional table": lambda rel: orc.relative_position_bucket(rel, True, NB, MD),
    }


@pytest.mark.parametrize("round_scores", [False, True])
@pytest.mark.parametrize("T", [1, 2, 16, 17, 33, 128, 129, 256])
@pytest.mark.parametrize("H", [64, 32])
def test_t5_decoder_self_attn_scoring_kernel(ops, H, T, round_scores):
    """The scoring path's kernel at every T it allows (up to 256: the exact buckets, the log buckets, the saturation at 128)."""
    gen = torch.Generator(device="cuda").manual_seed(T * 7 + H)
    B = 2
    qkv = t5_data((B * T, 3 * H * 64), gen)
    rel_emb = t5_rel_emb(H, gen)
    out = ops.t5_decoder_self_attn(qkv, B, T, H, rel_emb, t5_lut(ops), MD, round_scores).float().view(B, T, H, 64)
    torch.cuda.synchronize()
    x = qkv.view(B, T, 3, H, 64)
    vmax = float(x[:, :, 2].float().abs().max())
    moved = {w: 0.0 for w in t5_mistakes()}
    for b in range(B):
        for tq in range(T):
            ref = ref_t5_row(x[b, tq, 0], x[b, :tq + 1, 1], x[b, :tq + 1, 2], tq, rel_emb, round_scores)
            tol = t5_tolerance(ref, vmax)
            err = (out[b, tq].double() - ref).abs()
            assert bool((err <= tol).all()), (b, tq, float(err.max()))
            if tq in (T - 1, T // 2) and tq > 0:
                for what, fn in t5_mistakes().items():
                    wrong = ref_t5_row(x[b, tq, 0], x[b, :tq + 1, 1], x[b, :tq + 1, 2], tq, rel_emb, round_scores, buckets=fn)
                    moved[what] = max(moved[what], float(((wrong - ref).abs() / tol).max()))
    if T >= 17:     # below that every key is in an exact bucket shared by both tables; a shifted bucket still moves
        assert all(m > 1.0 for m in moved.values()), moved
    elif T >= 2:
        assert moved["bucket shifted by one"] > 1.0, moved


def fill_t5_cache(kc, vc, k_rows, v_rows):
    """k_rows / v_rows: per sequence [t, H, 64] -> slots 0..t - 1 of the cache [B, H, cap, 64] (the rest keeps the sentinel)."""
    for b, (kr, vr) in enumerate(zip(k_rows, v_rows)):
        t = kr.shape[0]
        kc.t[b, :, :t] = kr.transpose(0, 1)
        vc.t[b, :, :t] = vr.transpose(0, 1)


def expected_t5_cache(kc_before, k_new, slots):
    exp = kc_before.clone()
    for b, t in enumerate(slots):
        exp[b, :, t] = k_new[b].view(torch.int16)
    return exp


@pytest.mark.parametrize("round_scores", [False, True])
@pytest.mark.parametrize("H", [64, 32])
def test_t5_cached_self_attn_is_the_scoring_kernel_row_for_row(ops, H, round_scores):
    """Cache slots 0..t - 1 hold the K / V rows of a scoring sequence, row t is the step's input with lengths[b] = t (a different t per
    sequence in one launch): the cached kernel's output must be bit-identical to row t of the scoring kernel, and the append must have
    written exactly slot t."""
    gen = torch.Generator(device="cuda").manual_seed(H + round_scores)
    T, cap = 256, 2048
    ts = [0, 1, 15, 16, 17, 128, 200, 255]
    B = len(ts)
    qkv = t5_data((B * T, 3 * H * 64), gen)
    rel_emb = t5_rel_emb(H, gen)
    lut = t5_lut(ops)
    scoring = ops.t5_decoder_self_attn(qkv, B, T, H, rel_emb, lut, MD, round_scores).view(B, T, H * 64)
    x = qkv.view(B, T, 3, H, 64)
    kc, vc = Guarded((B, H, cap, 64)), Guarded((B, H, cap, 64))
    fill_t5_cache(kc, vc, [x[b, :t, 1] for b, t in enumerate(ts)], [x[b, :t, 2] for b, t in enumerate(ts)])
    k_before, v_before = kc.bits().clone(), vc.bits().clone()
    step = torch.stack([qkv.view(B, T, -1)[b, t] for b, t in enumerate(ts)]).contiguous()
    lengths = torch.tensor(ts, dtype=torch.int32, device="cuda")
    out = ops.t5_decode_self_attn(step, kc.t, vc.t, lengths, rel_emb, lut, MD, round_scores)
    torch.cuda.synchronize()
    want = torch.stack([scoring[b, t] for b, t in enumerate(ts)])
    assert torch.equal(out, want), [int((out[b] != want[b]).sum()) for b in range(B)]
    assert torch.equal(kc.bits(), expected_t5_cache(k_before, [x[b, t, 1] for b, t in enumerate(ts)], ts))
    assert torch.equal(vc.bits(), expected_t5_cache(v_before, [x[b, t, 2] for b, t in enumerate(ts)], ts))
    assert kc.guards_intact() and vc.guards_intact()


@pytest.mark.parametrize("round_scores", [False, True])
@pytest.mark.parametrize("H", [64, 32])
def test_t5_cached_self_attn_long_generations(ops, H, round_scores):
    """Positions up to 2047 of a cap = 2048 cache against the fp64 reference: the exact buckets, the log buckets and the saturation at
    |rel| >= 128 that a long generation reaches. lengths[b] = cap (a sequence finished by length) is clamped to position cap - 1: it
    writes slot cap - 1 only, with the guards intact."""
    gen = torch.Generator(device="cuda").manual_seed(3 * H + round_scores)
    cap = 2048
    lengths_list = [2047, 1500, 1000, 300, 160, 129, 128, 127, 5, 0, cap]
    pos = [min(L, cap - 1) for L in lengths_list]
    B = len(pos)
    rel_emb = t5_rel_emb(H, gen)
    k_hist = [t5_data((t, H, 64), gen) for t in pos]
    v_hist = [(torch.randn(t, H, 64, generator=gen, device="cuda")).bfloat16() for t in pos]
    step = t5_data((B, 3 * H * 64), gen)
    step.view(B, 3, H, 64)[:, 2] = torch.randn(B, H, 64, generator=gen, device="cuda").bfloat16()
    kc, vc = Guarded((B, H, cap, 64)), Guarded((B, H, cap, 64))
    fill_t5_cache(kc, vc, k_hist, v_hist)
    k_before, v_before = kc.bits().clone(), vc.bits().clone()
    lengths = torch.tensor(lengths_list, dtype=torch.int32, device="cuda")
    out = ops.t5_decode_self_attn(step, kc.t, vc.t, lengths, rel_emb, t5_lut(ops), MD, round_scores).float().view(B, H, 64)
    torch.cuda.synchronize()
    s = step.view(B, 3, H, 64)
    assert torch.equal(kc.bits(), expected_t5_cache(k_before, list(s[:, 1]), pos))
    assert torch.equal(vc.bits(), expected_t5_cache(v_before, list(s[:, 2]), pos))
    assert kc.guards_intact() and vc.guards_intact()
    moved = {w: 0.0 for w in t5_mistakes()}
    for b, t in enumerate(pos):
        k = torch.cat([k_hist[b], s[b, 1][None]])
        v = torch.cat([v_hist[b], s[b, 2][None]])
        vmax = float(v.float().abs().max())
        ref = ref_t5_row(s[b, 0], k, v, t, rel_emb, round_scores)
        tol = t5_tolerance(ref, vmax)
        err = (out[b].double() - ref).abs()
        assert bool((err <= tol).all()), (lengths_list[b], float(err.max()), float((err / tol).max()))
        if t >= 128:
            for what, fn in t5_mistakes().items():
                wrong = ref_t5_row(s[b, 0], k, v, t, rel_emb, round_scores, buckets=fn)
                moved[what] = max(moved[what], float(((wrong - ref).abs() / tol).max()))
    assert all(m > 1.0 for m in moved.values()), moved
