"""`-m gpu` checks of the head-dim-40 flash attention, which runs 192-query tiles (three consumer warpgroups of 64
rows): torch fp32 references at query counts that are and are not multiples of the tile, self / gated / cross key
sets, with and without the instance-isolation mask, in both storage builds; a ragged last tile writes nothing past
nq; launches are bitwise reproducible and a CUDA-graph replay equals the eager call."""
import pytest
import torch

pytestmark = pytest.mark.gpu

H, D = 8, 40
C = H * D
N_OBJ = 184  # UniFusion object tokens of the gated self-attention
N_CTX = 77   # text tokens of the cross-attention
NQS = (4096, 64, 100, 191, 193, 1000)
DTYPES = {"fp16": torch.float16, "bf16": torch.bfloat16}
# |err| <= REL * max|ref| + ABS: P and O are rounded to the storage type (bf16 has 8 significand bits, fp16 11)
TOL = {"fp16": (4e-3, 2e-3), "bf16": (3e-2, 1.6e-2)}


@pytest.fixture(params=list(DTYPES))
def storage(request, cuda_device):
    from instancediffusion_b200 import ops
    with ops.storage(DTYPES[request.param]):
        yield request.param


def _inputs(kind, B, nq, masked, dt, device, seed=0):
    g = torch.Generator().manual_seed(seed)
    n0 = N_CTX if kind == "cross" else nq
    n1 = N_OBJ if kind == "gated" else 0
    q = torch.randn((B * nq, C), generator=g).to(device, dt)
    kv0 = torch.randn((B * n0, 2 * C), generator=g).to(device, dt)
    kv1 = torch.randn((B * max(n1, 1), 2 * C), generator=g).to(device, dt)
    mask = None
    if masked:
        mq = torch.randint(0, 64, (B, nq), generator=g, dtype=torch.int64)
        mq = (mq & torch.randint(0, 64, (B, nq), generator=g, dtype=torch.int64)).to(torch.int32)  # sparse bits
        mk = torch.cat([mq, torch.randint(0, 64, (B, n1), generator=g, dtype=torch.int64).to(torch.int32)], 1)
        mask = (mq.to(device).contiguous(), mk.to(device).contiguous())
    return dict(q=q, kv0=kv0, kv1=kv1, n0=n0, n1=n1, mask=mask)


def _run(x, B, nq, out=None):
    from instancediffusion_b200 import ops
    kw = dict(k1=x["kv1"][:, :C], v1=x["kv1"][:, C:], n1=x["n1"], kv1_batch=B) if x["n1"] else {}
    if x["mask"] is not None:
        kw["mask"] = x["mask"]
    return ops.attention(x["q"], x["kv0"][:, :C], x["kv0"][:, C:], batch=B, heads=H, head_dim=D, nq=nq, n0=x["n0"],
                         scale=D ** -0.5, out=out, **kw)


def _reference(x, B, nq):
    n0, n1 = x["n0"], x["n1"]
    ref = torch.empty((B, nq, C), device=x["q"].device)
    for b in range(B):
        q = x["q"][b * nq:(b + 1) * nq].float().view(nq, H, D).transpose(0, 1)
        kv = x["kv0"][b * n0:(b + 1) * n0].float()
        if n1:
            kv = torch.cat([kv, x["kv1"][b * n1:(b + 1) * n1].float()], 0)
        k = kv[:, :C].reshape(-1, H, D).transpose(0, 1)
        v = kv[:, C:].reshape(-1, H, D).transpose(0, 1)
        s = (q @ k.transpose(-1, -2)) * D ** -0.5
        if x["mask"] is not None:
            mq, mk = x["mask"]
            allowed = (mq[b][:, None] & mk[b][None, :]) != 0
            idx = torch.arange(nq, device=s.device)
            allowed[idx, idx] = True  # a visual token always sees itself
            s = s.masked_fill(~allowed[None], float("-inf"))
        ref[b] = (torch.softmax(s, -1) @ v).transpose(0, 1).reshape(nq, C)
    return ref.view(B * nq, C)


def _check(out, ref, storage, what):
    rel, ab = TOL[storage]
    err = (out.float() - ref).abs().max().item()
    assert torch.isfinite(out.float()).all(), what
    assert err <= rel * ref.abs().max().item() + ab, f"{what}: max |err| {err:.3e}"


@pytest.mark.parametrize("B", [1, 8])
@pytest.mark.parametrize("nq", NQS)
@pytest.mark.parametrize("kind", ["self", "gated", "cross"])
def test_d40_vs_torch(storage, cuda_device, kind, nq, B):
    x = _inputs(kind, B, nq, False, DTYPES[storage], cuda_device)
    _check(_run(x, B, nq), _reference(x, B, nq), storage, f"{kind} B{B} nq{nq} {storage}")


# the mask is applied where the gated self-attention uses it: n0 = nq and n0 + n1 both multiples of 4
@pytest.mark.parametrize("B", [1, 8])
@pytest.mark.parametrize("nq", [n for n in NQS if n % 4 == 0])
@pytest.mark.parametrize("kind", ["self", "gated"])
def test_d40_masked_vs_torch(storage, cuda_device, kind, nq, B):
    x = _inputs(kind, B, nq, True, DTYPES[storage], cuda_device, seed=1)
    _check(_run(x, B, nq), _reference(x, B, nq), storage, f"masked {kind} B{B} nq{nq} {storage}")


@pytest.mark.parametrize("nq", [64, 100, 193, 1000])
def test_ragged_tile_writes_nothing_past_nq(cuda_device, nq):
    """The output is a column window of a wider buffer with spare rows after it: every element outside the
    window keeps its sentinel, so no row past nq and no column outside the heads is written."""
    B = 2
    x = _inputs("gated", B, nq, False, torch.float16, cuda_device, seed=2)
    sentinel = -1234.0
    buf = torch.full((B * nq + 256, C + 16), sentinel, dtype=torch.float16, device=cuda_device)
    out = buf[:B * nq, 8:8 + C]
    _run(x, B, nq, out=out)
    torch.cuda.synchronize()
    assert bool((buf[B * nq:] == sentinel).all()), "rows past batch * nq were written"
    assert bool((buf[:, :8] == sentinel).all()) and bool((buf[:, 8 + C:] == sentinel).all()), "columns outside the heads were written"
    _check(out, _reference(x, B, nq), "fp16", f"strided out nq{nq}")


@pytest.mark.parametrize("masked", [False, True])
def test_two_launches_are_bitwise_identical(cuda_device, masked):
    B, nq = 8, 4096
    x = _inputs("gated", B, nq, masked, torch.float16, cuda_device, seed=3)
    a = _run(x, B, nq).clone()
    b = _run(x, B, nq)
    assert torch.equal(a, b)


def test_graph_replay_equals_eager(cuda_device):
    B, nq = 8, 1000
    x = _inputs("gated", B, nq, True, torch.float16, cuda_device, seed=4)
    eager = _run(x, B, nq).clone()
    out = torch.empty_like(eager)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        _run(x, B, nq, out=out)  # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        _run(x, B, nq, out=out)
    out.zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, eager)
