"""GPU (-m gpu): the load pipeline of the tensor-core GQA decode kernel.

The kernel streams K through a ring of (Q, K) stages and V through a ring of V stages, freed at different points, and
prefetches the rows of items a few places ahead into L2.  These tests drive what those could break: many items per CTA
(both rings wrap many times), empty splits between full ones, a last split of one token, page sizes 16 / 32 / 64,
groups of 1, 4, 16 and 24 query heads (one real column of 16 up to a second block of 16 partly real), and a
speculative case.  Each case checks the oracle, that a request's rows do not depend on the rest of the batch (its CTA,
ring slots and prefetch neighbours change), and that a shuffled page table and the packed NHD view give the bits of the
contiguous cache."""
import math

import pytest
import torch

import gqa_spec_oracle as SO

pytestmark = pytest.mark.gpu

D = 128


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs an H100")
    return torch.device("cuda:0")


def _cos_diff(a, b):
    a, b = a.double().flatten(), b.double().flatten()
    return 1 - 2 * (a * b).sum() / max((a * a + b * b).sum(), 1e-12)


def _lens(B, S, kind):
    if kind == "full":
        return [S] * B
    if kind == "uneven":   # short requests leave empty splits between the full ones of their neighbours
        return [S if b % 3 == 0 else max(1, (S * (b % 7)) // 9 + b % 5) for b in range(B)]
    assert kind == "one_token_tail"   # the last split of every request holds one token
    return [max(1, (S - 1) // 128 - b % 3) * 128 + 1 for b in range(B)]


# (B, S, page, Hq, Hkv, Q, lens)
CASES = [
    (64, 2048, 16, 32, 8, 1, "full"),             # the Mixtral decode shape: 62 items per CTA
    (48, 1500, 16, 32, 8, 1, "uneven"),
    (40, 1100, 32, 8, 8, 1, "one_token_tail"),    # group 1: one real column of 16
    (24, 900, 64, 64, 4, 1, "uneven"),            # group 16
    (20, 1000, 16, 48, 2, 1, "one_token_tail"),   # group 24: N = 32, the second block of 16 partly real
    (16, 700, 32, 32, 8, 3, "uneven"),            # speculative decode, 3 draft tokens
]


def _decode(q, kc, vc, lens, pt, Q):
    from lvllm_b200 import ops
    out, lse = ops.gqa_decode(q, kc, vc, lens, pt, D ** -0.5, q_len_per_req=Q)
    torch.cuda.synchronize()
    return out.cpu(), lse.cpu()


def _same_bits(a, b):
    return torch.equal(a[0].view(torch.int16), b[0].view(torch.int16)) and torch.equal(a[1].view(torch.int32),
                                                                                      b[1].view(torch.int32))


@pytest.mark.parametrize("B,S,page,hq,hkv,Q,kind", CASES)
def test_pipeline(dev, B, S, page, hq, hkv, Q, kind):
    g = torch.Generator().manual_seed(B * 1000 + page)
    lens = torch.tensor(_lens(B, S, kind), dtype=torch.int32)
    npg = -(-S // page)
    pages = B * npg
    dgen = torch.Generator(device=dev).manual_seed(B + page)
    # the contiguous cache: request b owns pages [b * npg, (b + 1) * npg) in order
    kv = torch.randn(pages, page, hkv, 2 * D, generator=dgen, device=dev).bfloat16()   # packed NHD
    k_lin, v_lin = kv[..., :D].contiguous(), kv[..., D:].contiguous()
    pt_lin = torch.arange(pages, dtype=torch.int32).reshape(B, npg)
    q = torch.randn(B * Q, hq, D, generator=g).bfloat16().to(dev)
    lens_d = lens.to(dev)
    base = _decode(q, k_lin, v_lin, lens_d, pt_lin.to(dev), Q)
    out, lse = base
    assert not torch.isnan(out.float()).any() and not torch.isnan(lse).any()

    # oracle on the first, a middle and the last requests
    reqs = sorted({0, B // 2, B - 1})
    rows = [b * Q + i for b in reqs for i in range(Q)]
    sub = pt_lin[reqs]
    idx = sub.flatten().long().to(dev)
    ref, lse_ref = SO.gqa_decode(q[rows].cpu(), k_lin[idx].cpu(), v_lin[idx].cpu(), lens[reqs],
                                 torch.arange(sub.numel(), dtype=torch.int32).reshape(sub.shape), D ** -0.5, q_len=Q)
    assert _cos_diff(out.float()[rows], ref) < 1e-5
    torch.testing.assert_close(lse[rows], lse_ref, atol=1e-3, rtol=1e-3)

    # a request decoded alone (same page-table width, so the same splits) gives the bits it gets inside the batch
    for b in reqs:
        alone = _decode(q[b * Q:(b + 1) * Q], k_lin, v_lin, lens_d[b:b + 1], pt_lin[b:b + 1].to(dev), Q)
        r = slice(b * Q, (b + 1) * Q)
        assert _same_bits(alone, (out[r], lse[r])), f"request {b} alone differs from its rows in the batch"

    # the same keys and values on shuffled pages
    perm = torch.randperm(pages, generator=g)
    k_perm, v_perm = torch.empty_like(k_lin), torch.empty_like(v_lin)
    k_perm[perm.to(dev)], v_perm[perm.to(dev)] = k_lin, v_lin
    pt_perm = perm[pt_lin.long()].int()
    assert _same_bits(_decode(q, k_perm, v_perm, lens_d, pt_perm.to(dev), Q), base)

    # the packed NHD view, read through its strides
    assert _same_bits(_decode(q, kv[..., :D], kv[..., D:], lens_d, pt_lin.to(dev), Q), base)


def test_empty_requests_between_full_ones(dev):
    """Requests with one key next to long ones: most of a CTA's items are empty splits, which every role must skip alike."""
    B, S, page, hq, hkv = 33, 1024, 16, 32, 8
    g = torch.Generator().manual_seed(7)
    lens = torch.tensor([S if b % 4 == 0 else 1 for b in range(B)], dtype=torch.int32)
    npg = S // page
    k = torch.randn(B * npg, page, hkv, D, generator=g).bfloat16()
    v = torch.randn(B * npg, page, hkv, D, generator=g).bfloat16()
    pt = torch.randperm(B * npg, generator=g).reshape(B, npg).int()
    q = torch.randn(B, hq, D, generator=g).bfloat16()
    out, lse = _decode(q.to(dev), k.to(dev), v.to(dev), lens.to(dev), pt.to(dev), 1)
    ref, lse_ref = SO.gqa_decode(q, k, v, lens, pt, D ** -0.5)
    assert _cos_diff(out.float(), ref) < 1e-5
    torch.testing.assert_close(lse, lse_ref, atol=1e-3, rtol=1e-3)
    assert not math.isnan(float(out.float().sum()))
