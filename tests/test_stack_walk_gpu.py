"""H100: the Transformer stack's backward hands each layer's gradients over as soon as they are final, in both
residual modes."""
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _stack(streams):
    from audiolm_pytorch_b200.transformer import Transformer

    torch.manual_seed(0)
    return Transformer(dim=128, depth=3, heads=2, flash_attn=True, num_residual_streams=streams).to(DEV).train()


@pytest.mark.parametrize("streams", [1, 4])
def test_grad_ready_hook_fires_per_layer(streams):
    """with direct accumulation into `.grad` (parallel.FlatGradBucket.attach), grad_ready_hook(i) fires once per
    layer, top layer first; the gradients are then in `.grad`.  Without it autograd receives the gradients and the
    hook stays silent."""
    tr = _stack(streams)
    fired = []
    tr.grad_ready_hook = fired.append
    x = torch.randn(2, 64, 128, device=DEV)
    w = torch.randn(2, 64, 128, device=DEV)

    tr.accumulate_into_grad = True
    for p in tr.parameters():
        p.grad = torch.zeros_like(p)
    (tr(x).float() * w).sum().backward()
    assert fired == [2, 1, 0]
    assert all(torch.isfinite(p.grad).all() for p in tr.parameters())
    assert all(p.grad.abs().sum() > 0 for name, p in tr.named_parameters() if name.endswith(".weight"))

    fired.clear()
    tr.accumulate_into_grad = False
    (tr(x).float() * w).sum().backward()
    assert fired == []
