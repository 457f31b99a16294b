"""Fused gate + routing kernels, column sums and the public column scan against plain PyTorch fp32 references
(csrc/gate_route.cu; run with `pytest -m gpu` on an H100)."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def C():
    from tutel_b200.ops import backend
    return backend.require_ext()


def _torch_gate(logits, k, normalize):
    """Op-by-op reference: softmax, top-k, normalised gates, GShard loss (tutel/impls/fast_dispatch.py:143-176)."""
    S, E = logits.shape
    p = torch.softmax(logits.float(), dim=1)
    top, idx = torch.topk(p, k, dim=1)
    gates = top
    if normalize and k > 1:
        gates = top / torch.clamp(top.sum(dim=1, keepdim=True), min=float(torch.finfo(logits.dtype).eps))
    ce = torch.bincount(idx[:, 0], minlength=E).float()
    l_aux = (p.sum(0) * ce).sum() * (E / float(S * S))
    return p, idx, top, gates, l_aux


def _torch_locations(idx_ks, E):
    """Stable queue positions: all first choices in token order, then all second choices, ... """
    k, S = idx_ks.shape
    flat = idx_ks.reshape(-1).long()
    onehot = F.one_hot(flat, E)
    pos = torch.cumsum(onehot, dim=0) - 1
    return pos.gather(1, flat.unsqueeze(1)).view(k, S), onehot.sum(0)


@pytest.mark.parametrize('S,E,k,dtype', [(8192, 8, 2, torch.bfloat16), (777, 130, 4, torch.float32),
                                         (1000, 64, 1, torch.float16), (300, 512, 8, torch.float32)])
def test_gate_route_forward_matches_torch(C, S, E, k, dtype):
    torch.manual_seed(3)
    logits = (torch.randn(S, E, device='cuda') * 2).to(dtype)
    cap = k * ((S + E - 1) // E)
    scores, idx, top, gates, loc, counts, ce, l_aux, slot = C.gate_route_forward(logits, k, cap, True, float(torch.finfo(dtype).eps))
    p, ridx, rtop, rgates, rl = _torch_gate(logits, k, True)
    assert torch.allclose(scores, p, atol=2e-6)
    # ties between equal scores may be ordered differently by torch.topk: compare the selected VALUES, and ids where unique
    assert torch.allclose(top.t(), rtop, atol=2e-6)
    same = idx.t().long() == ridx
    assert same.float().mean() > 0.995
    assert torch.allclose(gates.t(), rgates, atol=1e-5, rtol=1e-4)
    assert torch.allclose(l_aux.float(), rl, rtol=2e-2 if dtype != torch.float32 else 1e-4)
    # routing of the kernel's own choices
    rloc, rcounts = _torch_locations(idx, E)
    assert torch.equal(loc.long(), rloc) and torch.equal(counts.long(), rcounts)
    assert torch.equal(ce, torch.bincount(idx[0].long(), minlength=E).float())
    # the inverse map: slot (e, l) -> token * k + choice, -1 where empty
    want = torch.full([E * cap], -1, dtype=torch.int32, device='cuda')
    valid = loc < cap
    tok = torch.arange(S, device='cuda', dtype=torch.int32).unsqueeze(0) * k + torch.arange(k, device='cuda', dtype=torch.int32).unsqueeze(1)
    want[(idx.long() * cap + loc.long())[valid]] = tok[valid]
    assert torch.equal(slot, want)


@pytest.mark.parametrize('E,k,normalize,dtype', [(8, 2, True, torch.bfloat16), (130, 4, True, torch.float32),
                                                (64, 3, False, torch.float32), (16, 1, True, torch.float16)])
def test_gate_route_autograd_matches_torch_autograd(E, k, normalize, dtype):
    """One-launch backward (normalisation + top-k selection + softmax + loss) vs autograd of the op-by-op formulation."""
    from tutel_b200.ops.gating import fused_gate_route
    torch.manual_seed(6)
    S = 1111
    base = torch.randn(S, E, device='cuda').to(dtype)
    wg = torch.randn(k, S, device='cuda')
    a = base.clone().requires_grad_(True)
    idx, loc, gates, l_aux, counts, top1, slot = fused_gate_route(a, k, normalize, 0)
    ((gates * wg).sum() + 2.0 * l_aux.float()).backward()
    b = base.float().clone().requires_grad_(True)
    p = torch.softmax(b, dim=1)
    rtop = p.gather(1, idx.t().long())                       # same selection as the kernel
    rg = rtop / torch.clamp(rtop.sum(1, keepdim=True), min=float(torch.finfo(dtype).eps)) if (normalize and k > 1) else rtop
    ce = torch.bincount(idx[0].long(), minlength=E).float()
    rl = (p.sum(0) * ce).sum() * (E / float(S * S))
    ((rg.t() * wg).sum() + 2.0 * rl).backward()
    tol = 1e-5 if dtype == torch.float32 else 2e-2
    assert slot is None and torch.allclose(gates, rg.t(), atol=1e-5)
    assert torch.allclose(a.grad.float(), b.grad, atol=tol * b.grad.abs().max().item() + 1e-7, rtol=tol)


def test_layer_fused_gate_matches_op_by_op(monkeypatch):
    """The whole layer with the fused CUDA gate/route vs TUTEL_B200_FUSED_GATE=0 (fp32: tight tolerance)."""
    from tutel_b200 import moe
    outs = []
    for mode in ('0', 'auto'):
        monkeypatch.setenv('TUTEL_B200_FUSED_GATE', mode)
        torch.manual_seed(0)
        layer = moe.moe_layer(gate_type={'type': 'top', 'k': 2, 'capacity_factor': 1.25}, model_dim=64,
                              experts={'type': 'ffn', 'num_experts_per_device': 4, 'hidden_size_per_expert': 128,
                                       'activation_fn': lambda t: F.relu(t)}, seeds=(1, 1, 1)).cuda()
        x = torch.randn(6, 50, 64, device='cuda', requires_grad=True)
        y = layer(x)
        (y.pow(2).mean() + 0.1 * y.l_aux).backward()
        outs.append((y.detach(), y.l_aux.detach(), x.grad.clone(), layer.gates[0].wg.weight.grad.clone(),
                     layer.dispatch_count.clone()))
    for u, v in zip(outs[0], outs[1]):
        assert torch.allclose(u.float(), v.float(), atol=1e-5, rtol=1e-4)


@pytest.mark.parametrize('G,T,N,dtype', [(8, 2048, 4096, torch.bfloat16), (1, 333, 264, torch.float32),
                                         (3, 1000, 520, torch.float16), (2, 16384, 128, torch.bfloat16)])
def test_grouped_colsum(C, G, T, N, dtype):
    torch.manual_seed(5)
    x = torch.randn(G, T, N, device='cuda').to(dtype)
    out = C.grouped_colsum(x)
    ref = x.float().sum(dim=1)
    assert out.dtype == dtype and torch.allclose(out.float(), ref, atol=2e-2 * T ** 0.5 if dtype != torch.float32 else 1e-3, rtol=1e-2)
    xs = x[:, : T // 2]                                      # strided groups (a view)
    assert torch.allclose(C.grouped_colsum(xs).float(), xs.float().sum(dim=1), atol=2e-2 * T ** 0.5, rtol=1e-2)


@pytest.mark.parametrize('S,E', [(8192, 8), (1000, 130), (33, 1), (70000, 3), (4097, 2048)])
def test_fast_cumsum_sub_one(S, E):
    from tutel_b200 import moe
    torch.manual_seed(8)
    mask = (torch.rand(S, E, device='cuda') < 0.3).to(torch.int64)
    out = moe.fast_cumsum_sub_one(mask)
    assert torch.equal(out.long(), torch.cumsum(mask, dim=0) - 1)


@pytest.mark.parametrize('dtype,act', [(torch.float32, 'relu'), (torch.bfloat16, 'silu'), (torch.float16, 'gelu')])
def test_skinny_ffn_matches_torch(C, dtype, act):
    """Both expert layers in one weight-streaming launch vs fp32 torch (rows past the device-side counts stay zero)."""
    torch.manual_seed(9)
    G, R, K, H, N = 5, 12, 256, 200, 136
    x = torch.randn(G, R, K, device='cuda').to(dtype)
    w1 = (torch.randn(G, H, K, device='cuda') * 0.1).to(dtype)
    w2 = (torch.randn(G, H, N, device='cuda') * 0.1).to(dtype)
    b1, b2 = torch.randn(G, H, device='cuda').to(dtype), torch.randn(G, N, device='cuda').to(dtype)
    counts = torch.tensor([12, 0, 1, 9, 30], device='cuda', dtype=torch.int32)
    y = C.skinny_ffn(x, w1, b1, w2, b2, counts, {'relu': 1, 'gelu': 2, 'silu': 3}[act])
    fn = {'relu': F.relu, 'gelu': F.gelu, 'silu': F.silu}[act]
    ref = torch.matmul(fn(torch.matmul(x.float(), w1.float().transpose(1, 2)) + b1.float().unsqueeze(1)), w2.float()) + b2.float().unsqueeze(1)
    mask = (torch.arange(R, device='cuda').view(1, R, 1) < counts.clamp(max=R).view(G, 1, 1))
    ref = torch.where(mask, ref, torch.zeros((), device='cuda'))
    tol = 1e-4 if dtype == torch.float32 else 3e-2
    assert y.dtype == torch.float32 and torch.allclose(y, ref, atol=tol * 4, rtol=tol)


def test_dropless_layer_without_host_sync_matches_padded_path(monkeypatch):
    """capacity_factor=0 + megablocks_size=1 on one GPU: the worst-case row bound (no read-back of the capacity) gives the
    same output as the dense path with the exact dynamic capacity."""
    from tutel_b200 import moe
    torch.manual_seed(0)
    layer = moe.moe_layer(gate_type={'type': 'top', 'k': 2, 'capacity_factor': 0.0}, model_dim=256,
                          experts={'type': 'ffn', 'num_experts_per_device': 16, 'hidden_size_per_expert': 512,
                                   'activation_fn': lambda t: F.relu(t)}, seeds=(1, 1, 1)).cuda().eval()
    x = torch.randn(1, 24, 256, device='cuda')
    with torch.no_grad():
        dense = layer(x)
        fast = layer(x, megablocks_size=1)
    assert torch.allclose(dense, fast, atol=1e-4, rtol=1e-4)


@pytest.mark.parametrize('act', ['gelu', 'silu', 'relu'])
def test_fused_act_ffn_matches_autograd(act):
    """GELU / SiLU experts on the wgmma kernel: the forward epilogue also stores the pre-activation, the dgrad epilogue
    applies act'(pre) - checked against plain fp32 autograd."""
    from tutel_b200.ops import gemm as G
    torch.manual_seed(12)
    Gn, T, M, H = 2, 384, 256, 512
    x = (torch.randn(Gn, T, M, device='cuda') * 0.5).bfloat16().requires_grad_(True)
    w1 = (torch.randn(Gn, H, M, device='cuda') * 0.06).bfloat16().requires_grad_(True)
    w2 = (torch.randn(Gn, H, M, device='cuda') * 0.06).bfloat16().requires_grad_(True)
    b1 = (torch.randn(Gn, H, device='cuda') * 0.1).bfloat16().requires_grad_(True)
    b2 = (torch.randn(Gn, M, device='cuda') * 0.1).bfloat16().requires_grad_(True)
    y = G.fused_act_ffn(x, w1, b1, w2, b2, None, act)
    dy = torch.randn_like(y) * 0.1
    y.backward(dy)
    fn = {'relu': F.relu, 'gelu': F.gelu, 'silu': F.silu}[act]
    ps = [t.detach().float().requires_grad_(True) for t in (x, w1, b1, w2, b2)]
    yr = torch.matmul(fn(torch.matmul(ps[0], ps[1].transpose(1, 2)) + ps[2].unsqueeze(1)), ps[3]) + ps[4].unsqueeze(1)
    yr.backward(dy.float())

    def rel(a, b):
        return ((a.float() - b).norm() / b.norm()).item()
    errs = [rel(y, yr)] + [rel(t.grad, r.grad) for t, r in zip((x, w1, b1, w2, b2), ps)]
    assert max(errs) < 0.02, errs


def test_graphed_dropless_forward_matches_eager():
    """The bound-based dropless forward never touches the host, so it can be replayed as one CUDA graph."""
    from tutel_b200 import moe
    from tutel_b200.utils.graph import GraphedForward
    torch.manual_seed(1)
    layer = moe.moe_layer(gate_type={'type': 'top', 'k': 2, 'capacity_factor': 0.0}, model_dim=128,
                          experts={'type': 'ffn', 'num_experts_per_device': 32, 'hidden_size_per_expert': 256,
                                   'activation_fn': lambda t: F.relu(t)}, seeds=(1, 1, 1)).cuda().eval()
    xs = [torch.randn(1, 16, 128, device='cuda') for _ in range(3)]
    fast = GraphedForward(lambda t: layer(t, megablocks_size=1), xs[0])
    for x in xs:
        with torch.no_grad():
            want = layer(x, megablocks_size=1)
        got = fast(x).clone()
        assert torch.allclose(got, want, atol=1e-5, rtol=1e-5)


def test_quantize_transpose_matches_row_quantisation_of_the_transpose(C):
    """Transposing e4m3 quantisation of a weight == row quantisation of its 16-bit transpose (same scales, same bytes)."""
    torch.manual_seed(13)
    w = (torch.randn(3, 256, 192, device='cuda') * 0.3).bfloat16()
    qT, sT = C.quantize_transpose(w)
    q, s = C.quantize_rows(w.transpose(1, 2).contiguous())
    assert qT.shape == (3, 192, 256) and torch.allclose(sT, s, rtol=1e-6)
    assert torch.equal(qT.view(torch.uint8), q.view(torch.uint8))


def test_graphed_train_step_matches_eager_training():
    """zero_grad + forward + loss + backward + SGD of an MoE layer replayed as ONE CUDA graph: same loss trajectory as the
    eager loop (nothing in a single-GPU step touches the host)."""
    from tutel_b200 import moe
    from tutel_b200.utils.graph import GraphedTrainStep

    def build():
        torch.manual_seed(7)
        layer = moe.moe_layer(gate_type={'type': 'top', 'k': 2}, model_dim=256,
                              experts={'type': 'ffn', 'num_experts_per_device': 4, 'hidden_size_per_expert': 512,
                                       'activation_fn': lambda t: F.relu(t)}, seeds=(1, 1, 1)).cuda().to(torch.bfloat16)
        opt = torch.optim.SGD(layer.parameters(), lr=1e-2)

        def step(x, y):
            opt.zero_grad()
            x.grad = None
            out = layer(x)
            loss = F.mse_loss(out.float(), y) + layer.l_aux.float() * 0.01
            loss.backward()
            opt.step()
            return loss
        return step

    torch.manual_seed(11)
    xs = [torch.randn(2, 256, 256, device='cuda', dtype=torch.bfloat16) for _ in range(6)]
    ys = [torch.randn(2, 256, 256, device='cuda') for _ in range(6)]
    # Both twins first train eagerly on the default stream (the usual situation: a loop that is already running gets
    # captured).  The constructor then runs `warmup` real steps on the example inputs (the capture itself executes
    # nothing), so the eager twin takes the same step; from then on both see the same batches.
    eager, step = build(), build()
    for fn in (eager, step):
        for _ in range(2):
            fn(xs[0].clone().requires_grad_(True), ys[0])
    eager(xs[0].clone().requires_grad_(True), ys[0])
    want = [float(eager(x.clone().requires_grad_(True), y)) for x, y in zip(xs[1:], ys[1:])]
    fast = GraphedTrainStep(step, xs[0].clone().requires_grad_(True), ys[0], warmup=1)
    got = [float(fast(x, y)) for x, y in zip(xs[1:], ys[1:])]
    assert fast.launches_per_replay > 5
    for g, w in zip(got, want):
        assert abs(g - w) <= 1e-2 * abs(w), (got, want)
    assert fast.static_inputs[0].grad is not None and float(fast.static_inputs[0].grad.abs().sum()) > 0
