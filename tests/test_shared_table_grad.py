"""SharedTableGrad (neuralsim_b200/fields/fused_color.py): the boundary and colour backward nodes of the static step scatter into one
table gradient.  Both take the table through the holder's identity node (`route`), add their part into `take()` and return None; the
identity node hands the buffer on once both have run.  Checked here on CPU with toy nodes that write into the shared buffer as the
kernels do: the gradient is the sum of the parts in either order, when only one node is reached, with other contributors to the same
leaf, with two holders in one loss (two renders), and on every backward pass of a retained graph."""
import pytest
import torch

from neuralsim_b200.fields.fused_color import SharedTableGrad


class _Part(torch.autograd.Function):
    """y = sum(x) * k; backward adds k * g into the holder's buffer and returns None for x, as the static step's nodes do"""

    @staticmethod
    def forward(ctx, holder, k, x):
        ctx.holder, ctx.k, ctx.shape = holder, k, x.shape
        return (x * k).sum()

    @staticmethod
    def backward(ctx, g):
        ctx.holder.take(ctx.shape, g.device).add_(g * ctx.k)
        return None, None, None


def _two_nodes(x, holder, order):
    """3 * a + 7 * b with a = 2 sum(x), b = 5 sum(x): d/dx = 41.  The engine runs the node created later first: the creation order
    decides which node allocates the buffer."""
    t = holder.route(x)
    if order == "ab":
        a = _Part.apply(holder, 2.0, t)
        b = _Part.apply(holder, 5.0, t)
    else:
        b = _Part.apply(holder, 5.0, t)
        a = _Part.apply(holder, 2.0, t)
    return a * 3.0 + b * 7.0


@pytest.mark.parametrize("order", ["ab", "ba"])
def test_sum_of_both_parts(order):
    x = torch.randn(10, requires_grad=True)
    holder = SharedTableGrad()
    _two_nodes(x, holder, order).backward()
    assert torch.equal(x.grad, torch.full_like(x, 41.0)) and holder.buf is None


def test_one_node_reached():
    """a loss on one node's output only: its part alone"""
    x = torch.randn(10, requires_grad=True)
    holder = SharedTableGrad()
    t = holder.route(x)
    a = _Part.apply(holder, 2.0, t)
    _Part.apply(holder, 5.0, t)
    (a * 3.0).backward()
    assert torch.equal(x.grad, torch.full_like(x, 6.0)) and holder.buf is None


@pytest.mark.parametrize("where", ["before", "after"])
@pytest.mark.parametrize("order", ["ab", "ba"])
def test_other_contributors_to_the_leaf(order, where):
    """a plain term on the same leaf (a regulariser, another query of the table), created before or after the two nodes: autograd
    may add it to the leaf's gradient before either node has run, and both parts must still arrive"""
    x = torch.randn(10, requires_grad=True)
    other = (x * 11.0).sum() if where == "before" else None
    y = _two_nodes(x, SharedTableGrad(), order)
    if other is None:
        other = (x * 11.0).sum()
    (y + other).backward()
    assert torch.equal(x.grad, torch.full_like(x, 52.0))


@pytest.mark.parametrize("order", ["ab", "ba"])
def test_two_holders_in_one_loss(order):
    """two static renders in one loss (e.g. camera and LiDAR rays), each with its own holder"""
    x = torch.randn(10, requires_grad=True)
    (_two_nodes(x, SharedTableGrad(), order) + 2.0 * _two_nodes(x, SharedTableGrad(), "ba" if order == "ab" else "ab")).backward()
    assert torch.equal(x.grad, torch.full_like(x, 123.0))


def test_retained_graph_and_accumulation():
    """every backward pass starts from a fresh zeroed buffer; .grad accumulates the passes"""
    x = torch.randn(10, requires_grad=True)
    holder = SharedTableGrad()
    y = _two_nodes(x, holder, "ab")
    y.backward(retain_graph=True)
    assert torch.equal(x.grad, torch.full_like(x, 41.0))
    y.backward()
    assert torch.equal(x.grad, torch.full_like(x, 82.0)) and holder.buf is None
    g, = torch.autograd.grad(_two_nodes(x, holder, "ba"), [x])
    assert torch.equal(g, torch.full_like(x, 41.0))
