"""The fused VQ-GAN bottleneck attention on a range of query rows (rs_op_vq_attention_rows, rs_vq_set_attention_rows)
and the encode / decode passes split at that attention (rs_vq_*_begin / _end, VQModelTorch.attention_team).

Every comparison is torch.equal: a query row's result depends only on that row and on all keys and values, walked in
one fixed order, so the rows of several members, assembled, must be bit-identical to one full call."""
import ctypes as C

import pytest
import torch

from resshift_b200.parallel import attention_row_ranges
from resshift_b200.vq_arch import random_vq_state_dict, vq_preset

pytestmark = pytest.mark.gpu

SENTINEL = -1234.0


def _lib():
    from resshift_b200 import _lib
    return _lib


def _qkv(N, T, Cc, seed, ld):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return [torch.randn(N, T, ld, device="cuda", generator=g).half()[..., :Cc] for _ in range(3)]


def _rows(q, k, v, ld, rb, re, out):
    L = _lib()
    N, T, Cc = q.shape
    L.check(L.lib.rs_op_vq_attention_rows(q.data_ptr(), k.data_ptr(), v.data_ptr(), N, T, Cc, ld, rb, re, out.data_ptr(),
                                          L.current_stream()))


OP_CASES = [(c, t, n, c) for c in (128, 256, 512) for t in (16384, 65536) for n in (1, 2)] + [(256, 16384, 2, 384)]


@pytest.mark.parametrize("C_,T,N,ld", OP_CASES, ids=[f"C{c}-T{t}-N{n}-ld{ld}" for c, t, n, ld in OP_CASES])
def test_op_members_leave_other_rows_and_assemble_to_full(C_, T, N, ld):
    L = _lib()
    q, k, v = _qkv(N, T, C_, seed=C_ + T + N + ld, ld=ld)
    full = torch.empty(N, T, C_, dtype=torch.float16, device="cuda")
    L.check(L.lib.rs_op_vq_attention(q.data_ptr(), k.data_ptr(), v.data_ptr(), N, T, C_, ld, full.data_ptr(), L.current_stream()))
    assert torch.isfinite(full).all()
    for members in (2, 3, 7):
        assembled = torch.empty_like(full)
        for rb, re in attention_row_ranges(T, members):
            out = torch.full_like(full, SENTINEL)
            _rows(q, k, v, ld, rb, re, out)
            torch.cuda.synchronize()
            assert bool((out[:, :rb] == SENTINEL).all()) and bool((out[:, re:] == SENTINEL).all()), (members, rb, re)
            assembled[:, rb:re] = out[:, rb:re]
        assert torch.equal(assembled, full), (members, (assembled.float() - full.float()).abs().max().item())


def test_op_rejects_bad_ranges():
    L = _lib()
    q = torch.zeros(1, 16384, 128, dtype=torch.float16, device="cuda")
    out = torch.empty_like(q)
    for rb, re, msg in [(0, 0, "empty"), (64, 64, "empty"), (32, 128, "multiples of 64"), (0, 100, "multiples of 64"),
                        (0, 16384 + 64, "outside"), (-64, 64, "outside"), (128, 64, "outside")]:
        with pytest.raises(L.RsError, match=msg):
            _rows(q, q, q, 128, rb, re, out)


# ------------------------------------------------------------------------------------------------------------ plans

def _vq(name, seed=0):
    from resshift_b200.models.autoencoder import VQModelTorch
    cfg = vq_preset(name)
    m = VQModelTorch(**cfg.to_kwargs())
    m.load_state_dict(random_vq_state_dict(cfg, seed), strict=True)
    return cfg, m.cuda().eval()


def _team_runs(m, call, members, which):
    """Virtual members of a team, one after the other: each runs the pass inside attention_team, first to capture its
    own rows, then with every other member's captured rows written in by its exchange.  Returns the outputs of the
    second runs."""
    own = {}

    def capture(member):
        def exchange(view, rb, re):
            own[member] = view[:, rb:re].clone()
        return exchange

    def fill(member):
        def exchange(view, rb, re):
            assert torch.equal(view[:, rb:re], own[member])       # the member's own rows, as computed in the first run
            for m2, (b2, e2) in enumerate(attention_row_ranges(view.shape[1], members)):
                if m2 != member:
                    view[:, b2:e2] = own[m2]
        return exchange

    for member in range(members):
        with m.attention_team(member, members, capture(member)):
            call()
    outs = []
    for member in range(members):
        with m.attention_team(member, members, fill(member)):
            outs.append(call())
            ranges = attention_row_ranges(m.plan(which, *call.plan_key).attention.shape[1], members)
            assert m.attention_rows == [(which, *ranges[member])]
    return outs


def _check_encode(m, x, members_list=(2, 3, 8)):
    ref = m.encode(x).clone()
    enc = lambda: m.encode(x).clone()
    enc.plan_key = (x.shape[0], x.shape[2], x.shape[3])
    for members in members_list:
        for got in _team_runs(m, enc, members, 0):
            assert torch.equal(got, ref), members


def _check_decode(m, z, f, members_list=(2, 3, 8)):
    ref = m.decode(z).clone()
    ref_idx = m.last_indices.clone()

    def dec():
        out = m.decode(z).clone()
        assert torch.equal(m.last_indices, ref_idx)
        return out
    dec.plan_key = (z.shape[0], z.shape[2] * f, z.shape[3] * f)
    for members in members_list:
        for got in _team_runs(m, dec, members, 1):
            assert torch.equal(got, ref), members


def test_plan_f4_encode_1024():
    """f4 encode of a 1024x1024 image (T = 65536, C = 512)."""
    cfg, m = _vq("f4")
    x = torch.rand(1, 3, 1024, 1024, device="cuda", generator=torch.Generator(device="cuda").manual_seed(11)) * 2 - 1
    _check_encode(m, x)


def test_plan_f4_decode_256_latent():
    """f4 decode (quantised) of a 256x256 latent (T = 65536, C = 512): the image and the code indices."""
    cfg, m = _vq("f4")
    z = torch.randn(1, 3, 256, 256, device="cuda", generator=torch.Generator(device="cuda").manual_seed(12)) * 0.6
    _check_decode(m, z, cfg.downscale)


def test_plan_tiny_512x768_batch2():
    """tiny encode and decode at 512x768, batch 2 (a 128x192 bottleneck, T = 24576, C = 128)."""
    cfg, m = _vq("tiny", seed=2)
    g = torch.Generator(device="cuda").manual_seed(14)
    x = torch.rand(2, 3, 512, 768, device="cuda", generator=g) * 2 - 1
    z = torch.randn(2, 3, 128, 192, device="cuda", generator=g) * 0.6
    _check_encode(m, x)
    _check_decode(m, z, cfg.downscale)


def test_begin_end_equal_whole_pass_through_the_c_abi():
    """rs_vq_encode_begin + _end and rs_vq_decode_begin + _end (default rows) equal rs_vq_encode / rs_vq_decode."""
    L = _lib()
    cfg, m = _vq("tiny")
    g = torch.Generator(device="cuda").manual_seed(5)
    x = torch.rand(1, 3, 512, 512, device="cuda", generator=g) * 2 - 1
    ref = m.encode(x).clone()
    plan = m.plan(0, 1, 512, 512)
    out = torch.empty_like(ref)
    st = L.current_stream()
    L.check(L.lib.rs_vq_encode_begin(plan.handle, x.data_ptr(), st))
    L.check(L.lib.rs_vq_encode_end(plan.handle, out.data_ptr(), st))
    assert torch.equal(out, ref)
    img = m.decode(ref).clone()
    idx = m.last_indices.clone()
    plan = m.plan(1, 1, 512, 512)
    out, idx2 = torch.empty_like(img), torch.empty_like(idx)
    L.check(L.lib.rs_vq_decode_begin(plan.handle, ref.data_ptr(), idx2.data_ptr(), 0, st))
    L.check(L.lib.rs_vq_decode_end(plan.handle, out.data_ptr(), st))
    assert torch.equal(out, img) and torch.equal(idx2, idx)


def test_plan_row_calls_errors_and_description():
    L = _lib()
    cfg, m = _vq("f4")
    small = m.plan(0, 1, 256, 256)                     # 64x64 bottleneck: T = 4096, the GEMM + row-softmax form
    assert small.attention is None
    ptr, a, b, t, c = C.c_void_p(), C.c_longlong(), C.c_longlong(), C.c_int32(), C.c_int32()
    for rc in (L.lib.rs_vq_set_attention_rows(small.handle, 0, 4096),
               L.lib.rs_vq_attention_output(small.handle, C.byref(ptr), C.byref(a), C.byref(b), C.byref(t), C.byref(c))):
        with pytest.raises(L.RsError, match="no fused attention"):
            L.check(rc)
    # inside a team context, a plan without the fused attention runs as usual
    x = torch.rand(1, 3, 256, 256, device="cuda") * 2 - 1
    ref = m.encode(x).clone()
    with m.attention_team(1, 2, lambda *args: pytest.fail("no exchange without the fused attention")):
        assert torch.equal(m.encode(x), ref)
        assert m.attention_rows == []

    cfg, m = _vq("tiny")
    x = torch.rand(1, 3, 512, 512, device="cuda") * 2 - 1
    m.encode(x)
    plan = m.plan(0, 1, 512, 512)
    assert plan.attention.shape == (1, 16384, 128)
    for rb, re, msg in [(32, 64, "multiples of 64"), (0, 16384 + 64, "outside"), (128, 64, "outside"), (-64, 0, "outside")]:
        with pytest.raises(L.RsError, match=msg):
            L.check(L.lib.rs_vq_set_attention_rows(plan.handle, rb, re))

    def vq_attn_rows():
        cap, stride = 1024, 160
        ms = (C.c_double * cap)()
        desc = C.create_string_buffer(cap * stride)
        n = C.c_int32()
        L.check(L.lib.rs_vq_profile_ops(plan.handle, ms, desc, stride, cap, C.byref(n), L.current_stream()))
        rows = [desc.raw[i * stride:(i + 1) * stride].split(b"\0")[0].decode() for i in range(n.value)]
        return [r for r in rows if r.startswith("vq_attn")]

    L.check(L.lib.rs_vq_set_attention_rows(plan.handle, 5504, 11008))
    try:
        assert vq_attn_rows() == ["vq_attn T=16384 C=128 N=1 rows=5504:11008"]
    finally:
        L.check(L.lib.rs_vq_set_attention_rows(plan.handle, 0, 16384))
    assert vq_attn_rows() == ["vq_attn T=16384 C=128 N=1"]
    with pytest.raises(ValueError):
        with m.attention_team(2, 2, lambda *args: None):
            pass
