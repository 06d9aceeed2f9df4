"""The grouped wgmma GEMM and the MoE scatter / gather kernels against the float64 oracle of tests/gemm_oracle.py.

Sorts after the validated suites (see test_zz_new_kernels_gpu.py). Shapes follow the kernel's structure, derived from the SM
count of the device rather than hard-coded:

* both BN instantiations (BN = 256 when N % 256 == 0, else 128; STAGES = 4 or 6);
* ``num_kb = K / 64`` in {1, STAGES-1, STAGES, STAGES+1, 2·STAGES+3}: the stage ring's parity carried into a CTA's next tile at
  every phase;
* tile counts {1, SMs-1, SMs, SMs+1, > 3·SMs}: persistent CTAs with one, two and four tiles, so a stale accumulator shows;
* G in {1, 3, 8}, with and without bias, plain and GELU epilogue.

Integer data (every partial sum exact in fp32) must give the bits of the rounded float64 result; GELU and random data must
stay within :func:`gemm_oracle.gemm_bound`. References are float64 on the GPU.
"""
import pytest
import torch

from tests import gemm_oracle as go

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda", 0)


@pytest.fixture(scope="module")
def sms(dev):
    return torch.cuda.get_device_properties(dev).multi_processor_count


@pytest.fixture(scope="module")
def C():
    from bagua_b200.core import native

    return native()


def _num_kb(spec: str, BN: int) -> int:
    S = go.stages(BN)
    return {"1": 1, "S-1": S - 1, "S": S, "S+1": S + 1, "2S+3": 2 * S + 3}[spec]


def _tiles(spec: str, sms: int, per_m: int) -> int:
    """Tile count for a spec, a multiple of ``per_m`` (tiles per 128-row block: G · N / BN)."""
    target = {"1": 1, "SMs-1": sms - 1, "SMs": sms, "SMs+1": sms + 1, "3SMs+": 3 * sms + 1}[spec]
    return -(-target // per_m) * per_m


def _shape(G, N, tiles_spec, kb_spec, sms):
    BN = go.block_n(N)
    per_m = G * (N // BN)
    T = _tiles(tiles_spec, sms, per_m)
    return G, T // per_m * go.BM, N, _num_kb(kb_spec, BN) * go.BK


KB_SPECS = ["1", "S-1", "S", "S+1", "2S+3"]
# (G, N, tiles, num_kb): exact tile counts need G = 1 and N = BN (SMs - 1 may be prime)
INT_CASES = ([(1, N, "1", kb) for N in (128, 256) for kb in KB_SPECS]
             + [(1, N, "1", kb) for N in (384, 640, 1024) for kb in ("1", "S", "2S+3")]
             + [(1, N, t, kb) for N in (128, 256) for t in ("SMs-1", "SMs", "SMs+1", "3SMs+") for kb in ("S", "S+1", "2S+3")]
             + [(1, N, "3SMs+", "S+1") for N in (640, 1024)]
             + [(G, N, "1", "S+1") for G in (3, 8) for N in (384, 640, 1024)]
             + [(3, 256, "SMs+1", "2S+3"), (8, 640, "3SMs+", "S-1")])


def _id(case):
    return "G{}_N{}_tiles{}_kb{}".format(*case)


@pytest.mark.parametrize("case", INT_CASES, ids=_id)
def test_grouped_gemm_integer_data_is_bit_exact(dev, sms, case):
    from bagua_b200.ops.gemm import grouped_gemm_tn

    G, M, N, K = _shape(*case, sms)
    gen = torch.Generator(device=dev).manual_seed(INT_CASES.index(case))
    a, b, bias = go.int_operands(G, M, N, K, gen, dev)
    for bb in (bias, None):
        want = go.ref_gemm(a, b, bb).to(torch.bfloat16)
        out = grouped_gemm_tn(a, b, bb)
        bad = (out.view(torch.int16) != want.view(torch.int16)).sum().item()
        assert bad == 0, f"{(G, M, N, K)} bias={bb is not None}: {bad} of {out.numel()} elements differ in their bits"
        go.check_gemm(grouped_gemm_tn(a, b, bb, act="gelu"), a, b, bb, "gelu", what=f"gelu {(G, M, N, K)} bias={bb is not None}")


# random data: the integer grid thinned out, the shapes of the earlier fp32-reference test, K = 8192, and scales 2^±20
RANDOM_CASES = ([_id(c) for c in ((1, 128, "1", "S+1"), (1, 256, "1", "2S+3"), (3, 384, "1", "S"), (8, 1024, "1", "S-1"),
                                   (1, 128, "SMs+1", "2S+3"), (1, 256, "3SMs+", "S+1"), (1, 640, "3SMs+", "S+1"))]
                + ["G1_M128_N128_K64", "G2_M256_N384_K192", "G4_M1024_N512_K1024", "G4_M2048_N1024_K256", "G2_M256_N256_K8192",
                   "G1_M384_N640_K8192"])


def _random_shape(spec, sms):
    if "_M" in spec:
        G, M, N, K = (int(p[1:]) for p in spec.split("_"))
        return G, M, N, K
    G, N, t, kb = spec.split("_")
    return _shape(int(G[1:]), int(N[1:]), t[len("tiles"):], kb[len("kb"):], sms)


@pytest.mark.parametrize("scale", [1.0, 2.0 ** 20, 2.0 ** -20], ids=["x1", "x2^20", "x2^-20"])
@pytest.mark.parametrize("spec", RANDOM_CASES)
def test_grouped_gemm_random_data_within_the_float64_bound(dev, sms, spec, scale):
    from bagua_b200.ops.gemm import grouped_gemm_tn

    G, M, N, K = _random_shape(spec, sms)
    gen = torch.Generator(device=dev).manual_seed(5)
    a = (torch.randn(G, M, K, device=dev, generator=gen) * scale).to(torch.bfloat16)
    b = (torch.randn(G, N, K, device=dev, generator=gen) * (scale / K ** 0.5)).to(torch.bfloat16)
    bias32 = torch.randn(G, N, device=dev, generator=gen) * scale * scale
    for bb in (bias32, bias32.to(torch.bfloat16), None):
        for act in ("none", "gelu"):
            go.check_gemm(grouped_gemm_tn(a, b, bb, act=act), a, b, bb, act, what=f"{spec} x{scale} {act} bias={None if bb is None else bb.dtype}")


# ---- grouped_linear autograd --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("G,M,N,K", [(1, 128, 128, 64), (2, 256, 384, 192), (4, 1024, 512, 1024), (4, 2048, 1024, 256), (3, 256, 640, 128),
                                     (2, 384, 256, 320)])
@pytest.mark.parametrize("bias_dtype", [torch.bfloat16, torch.float32], ids=["bf16_bias", "fp32_bias"])
def test_grouped_linear_autograd_matches_float64(dev, monkeypatch, G, M, N, K, bias_dtype):
    """Forward and the x / w / bias gradients. K % 128 == 0 runs both backward GEMMs on the kernel, K % 128 == 64 runs them on
    torch.bmm (fp32 accumulation: reduced-precision reduction is switched off for the test). The bias gradient is summed in fp32
    and returned in the bias's own dtype."""
    from bagua_b200.ops.gemm import grouped_linear

    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_bf16_reduced_precision_reduction", False)
    gen = torch.Generator(device=dev).manual_seed(7)
    x = torch.randn(G, M, K, device=dev, generator=gen).to(torch.bfloat16).requires_grad_(True)
    w = (torch.randn(G, N, K, device=dev, generator=gen) / K ** 0.5).to(torch.bfloat16).requires_grad_(True)
    bias = torch.randn(G, N, device=dev, generator=gen).to(bias_dtype).requires_grad_(True)
    y = grouped_linear(x, w, bias)
    go.check_gemm(y, x.detach(), w.detach(), bias.detach(), what="forward")
    gy = torch.randn(G, M, N, device=dev, generator=gen).to(torch.bfloat16)
    y.backward(gy)
    go.check_gemm(x.grad, gy, w.detach().transpose(1, 2).contiguous(), what="dx")
    go.check_gemm(w.grad, gy.transpose(1, 2).contiguous(), x.detach().transpose(1, 2).contiguous(), what="dw")
    assert bias.grad.dtype == bias_dtype
    ref = gy.double().sum(1)
    err = M * 2 * go.U32 * gy.double().abs().sum(1)
    bound = err + go.HALF_ULP[bias_dtype] * (ref.abs() + err) + go.TINY[bias_dtype]
    worst = ((bias.grad.double() - ref).abs() / bound).max().item()
    assert worst <= 1.0, f"bias gradient ({bias_dtype}) off by {worst:.3g} x its bound"


# ---- grouped_gemm_tn_push on virtual worlds ------------------------------------------------------------------------------------------
def _world(P):
    from bagua_b200.parallel.virtual import VirtualPeerWorld

    return VirtualPeerWorld(P, torch.device("cuda", 0), timeout_s=20.0)


SENTINEL = 0xA5


@pytest.mark.parametrize("cap", [128, 384])
@pytest.mark.parametrize("P", [1, 2, 3, 4])
def test_grouped_gemm_push_is_bit_exact_on_every_owner(C, P, cap):
    """Owner r's GEMM rows are ordered [source s][slot]; the tile of source s lands in s's buffer at [r][g][slot]. Integer data:
    bit-exact at every (owner, source, group, slot); GELU within the bound; nothing written past the [P][G][cap][N] region."""
    w = _world(P)
    gen = torch.Generator().manual_seed(60 + P + cap)
    for G in (1, 3):
        for N in (256, 640):
            for K in (64, 320):
                region = P * G * cap * N * 2
                buf = w.alloc(region + 4096, fill=lambda r, t: t.fill_(SENTINEL))
                ops = [go.int_operands(G, P * cap, N, K, gen, w.device) for _ in range(P)]
                for act in ("none", "gelu"):
                    code = {"none": 0, "gelu": 1}[act]
                    w.launch_all(lambda r, st: C.grouped_gemm_tn_push(ops[r][0].data_ptr(), ops[r][1].data_ptr(), ops[r][2].data_ptr(), G, N, K, code,
                                                                      w.comms[r], buf.buf, 0, cap, st))
                    for s in range(P):
                        t = buf.tensors[s]
                        assert bool((t[region:] == SENTINEL).all()), f"P={P} cap={cap} G={G} N={N} K={K}: owner wrote past the region on rank {s}"
                        got = t[:region].view(torch.bfloat16).view(P, G, cap, N)
                        for r in range(P):
                            a, b, bias = ops[r]
                            a_s = a[:, s * cap:(s + 1) * cap]
                            what = f"P={P} cap={cap} G={G} N={N} K={K} {act}: owner {r} -> source {s}"
                            if act == "none":
                                assert torch.equal(got[r], go.ref_gemm(a_s, b, bias).to(torch.bfloat16)), what
                            else:
                                go.check_gemm(got[r], a_s, b, bias, "gelu", what=what)
    w.check()


# ---- moe_scatter / moe_gather on virtual worlds --------------------------------------------------------------------------------------
def _code(dtype):
    from bagua_b200.core import dtype_code

    return dtype_code(dtype)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
@pytest.mark.parametrize("P", [1, 2, 3, 4, 8])
def test_moe_scatter_gather_match_the_float64_oracle(C, P, dtype):
    """Rows of 1, 8 and 129 16-byte vectors (the last runs the kernels' v0 loop twice and reaches its tail guard), grids of one
    block and of 64 (fewer when P · 64 CTAs would not all be resident at once: the P kernels spin on each other's barriers).

    * scatter, with an fp32 ``scale`` (one multiply, one rounding) and without: bit-exact, unfilled slots zero;
    * gather from buffers filled by hand, pull layout ([source][expert][slot] on the owner) and local layout
      ([owner][expert][slot] on the source, what the GEMM push writes): ``picked`` bit-exact, the output bit-exact on integer rows
      with power-of-two weights and within :func:`gemm_oracle.gather_bound` on random rows, with and without weights."""
    w = _world(P)
    dev = w.device
    S, K, E_local, Cap = 96, 2, 2, 40
    per_vec = 16 // torch.empty(0, dtype=dtype).element_size()
    gen = torch.Generator().manual_seed(51 + P)
    eidx, sidx = go.routing(P, S, K, E_local, Cap, gen)
    eidx = [e.to(dev) for e in eidx]
    sidx = [s.to(dev) for s in sidx]
    valid = [(s >= 0) for s in sidx]
    owner = [e // E_local for e in eidx]
    el = [e % E_local for e in eidx]
    slot = [s.clamp_min(0) for s in sidx]
    for M in (per_vec, 8 * per_vec, 129 * per_vec):
        nbytes = P * E_local * Cap * M * torch.empty(0, dtype=dtype).element_size()
        buf = w.alloc(nbytes)
        numel = P * E_local * Cap * M
        for nblocks in (1, min(64, w.max_blocks_per_rank)):
            what = f"P={P} {dtype} M={M} nblocks={nblocks}"
            toks = [torch.randn(S, M, generator=gen).to(dtype).to(dev) for _ in range(P)]
            scales = [torch.rand(S, K, generator=gen).to(dev) for _ in range(P)]
            for scale in (scales, None):
                w.launch_all(lambda r, st: C.moe_scatter(w.comms[r], buf.buf, 0, toks[r].data_ptr(), eidx[r].data_ptr(), sidx[r].data_ptr(),
                                                         scale[r].data_ptr() if scale is not None else 0, S, K, M, E_local, Cap, _code(dtype), nblocks, st))
                want = torch.zeros(P, P, E_local, Cap, M, dtype=dtype, device=dev)     # [owner][source][expert][slot]
                for r in range(P):
                    v = valid[r]
                    rows = toks[r].unsqueeze(1).expand(S, K, M)[v]
                    want[owner[r][v], r, el[r][v], sidx[r][v]] = go.scatter_ref(rows, None if scale is None else scale[r][v].unsqueeze(-1))
                for o in range(P):
                    got = buf.view(o, dtype, numel).view(P, E_local, Cap, M)
                    assert torch.equal(got, want[o]), f"{what} scale={scale is not None}: owner {o} holds the wrong rows (unfilled slots must be zero)"
            for integer in (True, False):
                if integer:
                    prod = torch.randint(-64, 65, (P, P, E_local, Cap, M), generator=gen).to(dtype).to(dev)   # [owner][source][expert][slot]
                    wts = [torch.exp2(torch.randint(-3, 2, (S, K), generator=gen).float()).to(dev) for _ in range(P)]
                else:
                    prod = torch.randn(P, P, E_local, Cap, M, generator=gen).to(dtype).to(dev)
                    wts = [torch.rand(S, K, generator=gen).to(dev) for _ in range(P)]
                for local in (False, True):
                    for r in range(P):                                                  # rank r's buffer
                        layout = prod[:, r] if local else prod[r]
                        buf.view(r, dtype, numel).copy_(layout.reshape(-1))
                    for weights in (None, wts):
                        outs = [torch.full((S, M), float("nan"), dtype=dtype, device=dev) for _ in range(P)]
                        picked = [torch.full((S, K, M), float("nan"), dtype=dtype, device=dev) for _ in range(P)]
                        w.launch_all(lambda r, st: C.moe_gather(w.comms[r], buf.buf, 0, outs[r].data_ptr(), eidx[r].data_ptr(), sidx[r].data_ptr(),
                                                                weights[r].data_ptr() if weights is not None else 0, picked[r].data_ptr(), S, K, M,
                                                                E_local, Cap, _code(dtype), nblocks, st, local))
                        for r in range(P):
                            tag = f"{what} integer={integer} local={local} weights={weights is not None}: source {r}"
                            pw = torch.where(valid[r].unsqueeze(-1), prod[owner[r], r, el[r], slot[r]], torch.zeros((), dtype=dtype, device=dev))
                            assert torch.equal(picked[r], pw), f"{tag}: picked rows differ"
                            wr = None if weights is None else weights[r]
                            ref = go.gather_ref(pw, wr, valid[r])
                            if integer:
                                assert torch.equal(outs[r], ref.to(dtype)), f"{tag}: output differs from the rounded float64 sum"
                            else:
                                go.check_gather(outs[r], pw, wr, valid[r], what=tag)


# ---- malformed inputs on the GPU -----------------------------------------------------------------------------------------------------
def test_grouped_gemm_rejects_unsupported_shapes_and_mixed_devices_without_launching(dev, C):
    from bagua_b200.ops.gemm import grouped_gemm_tn

    def ab(G=2, M=128, N=256, K=64):
        return torch.zeros(G, M, K, dtype=torch.bfloat16, device=dev), torch.zeros(G, N, K, dtype=torch.bfloat16, device=dev)

    a, b = ab()
    flat = torch.zeros(2 * 128 * 64 + 8, dtype=torch.bfloat16, device=dev)
    cases = [
        ("M % 128", ab(M=192), None, "M % 128"),
        ("N % 128", ab(N=320), None, "N % 128"),
        ("K % 64", ab(K=96), None, "K % 64"),
        ("a misaligned", (flat[1:1 + 2 * 128 * 64].view(2, 128, 64), b), None, "a must be 16-byte aligned"),
        ("a on the GPU, b on the CPU", (a, b.cpu()), None, "b is on cpu"),
        ("b on the GPU, a on the CPU", (a.cpu(), b), None, "b is on cuda"),
        ("bias on the CPU", (a, b), torch.zeros(2, 256), "bias is on cpu"),
        ("bias of shape [N]", (a, b), torch.zeros(256, device=dev), "bias must be"),
    ]
    torch.cuda.synchronize()
    before = C.launch_count()
    for name, (x, y), bias, msg in cases:
        with pytest.raises(ValueError, match=msg):
            grouped_gemm_tn(x, y, bias)
    torch.cuda.synchronize()
    assert C.launch_count() == before, "a malformed call reached the kernel"
