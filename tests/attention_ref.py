"""fp64 attention references and the per-element bound the attention kernels are held to (head-dim-128 prefill attention in
test_gpu_qwen_kernels.py, head-dim-64 attention in test_gpu_attention_d64.py)."""
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
