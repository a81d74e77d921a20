"""The captured CUDA graphs the product replays, held bit-identical to the eager walks the launch audits check
(tests/engine_walks.py): if a replay equals the audited eager walk bit for bit, every replayed launch inherits that walk's
launch audit.

A replay can go wrong where an eager walk cannot: an input tensor rebound instead of copied into (the graph keeps reading
the captured one), a workspace that carries state from one replay to the next, a LoRA re-pack the captured pointers do not
see, the separate `accumulate=True` graph.  A tolerance test would pass most of these, so the comparison is through integer
views (NaN and -0.0 count).
"""
import pytest
import torch

import engine_walks as walks

pytestmark = pytest.mark.gpu

_BITS = {2: torch.int16, 4: torch.int32, 8: torch.int64}


def assert_bits_equal(got, want, what):
    g, w = got.reshape(-1).view(_BITS[got.element_size()]), want.reshape(-1).view(_BITS[want.element_size()])
    diff = g != w
    if diff.any():
        first = int(diff.nonzero()[0])
        raise AssertionError(f'{what}: {int(diff.sum())} of {diff.numel()} elements differ, first at flat index {first}: '
                             f'replay {got.reshape(-1)[first].item()!r}, eager {want.reshape(-1)[first].item()!r}')


def test_train_step_graph_matches_eager(cuda):
    _train_step_graph_matches_eager(2)


def test_train_step_graph_matches_eager_batch4(cuda):
    """the same at batch_size_per_gpu 4, per-sample concept-token positions"""
    _train_step_graph_matches_eager(4)


def _train_step_graph_matches_eager(B):
    """bench.py's training step at batch B (SD1.5 UNet at 64 x 64 + 12-layer CLIP, regulariser, shared flat state), three
    steps on different x0 / noise / t / masks / token ids.  In each step the same inputs run eager, then through the captured
    graph (step 1 captures the plain graph, step 2 replays it, step 3 captures the accumulate=True graph), each from the same
    gradient bytes; the loss and the whole flat gradient buffer (with the two logged scalars) must agree bit for bit.
    The bench optimiser step follows, so that every step runs on re-packed LoRA operands."""
    w = walks.build_train_sd15_full(use_graph=True, B=B)
    eng, state = w.eng, w.state
    for step, seed in enumerate((200, 201, 202), 1):
        batch = walks.train_sd15_full_inputs(w, seed)
        accumulate = step == 3
        start = state.grads.clone()
        runs = {}
        for graph in (False, True):
            state.grads.copy_(start)
            eng.use_train_graph = graph
            loss = eng.forward_backward(**batch, accumulate=accumulate)
            torch.cuda.synchronize()
            runs[graph] = (loss.clone(), state.grads.clone())
        assert eng.tgraph is not None and len(eng._tgraphs) == (2 if accumulate else 1)
        what = f'step {step} ({"accumulate, " if accumulate else ""}{"capture" if step != 2 else "replay"})'
        assert torch.isfinite(runs[False][0][0]), f'{what}: eager loss {runs[False][0]}'
        assert_bits_equal(runs[True][0], runs[False][0], f'{what}: loss_out')
        assert_bits_equal(runs[True][1], runs[False][1], f'{what}: state.grads')
        walks.train_optimizer_step(w)
    torch.cuda.synchronize()


def test_sampling_graph_matches_eager(cuda):
    """The 4-prompt validation call (SD1.5 UNet, CFG batch 8): the latents after every step of an eager call and of a
    graph call must agree bit for bit.  The first pair captures the graph; the second, on different prompt embeddings and
    latents, replays it on the same engine first, so that the per-prompt text K/V update (UNetEngine.update_text) runs
    between the capture and the replays, and repeats the call eager after it."""
    pipe, cond, neg, lat = walks.build_validation_sd15()
    g = torch.Generator().manual_seed(31)
    inputs = [(cond, neg, lat), (torch.randn(cond.shape, generator=g), torch.randn(neg.shape, generator=g),
                                 torch.randn(lat.shape, generator=g))]
    engines, graphs = set(), set()
    for call, order in enumerate(((False, True), (True, False)), 1):
        runs = {}
        for graph in order:
            pipe.unet.use_graph = graph
            steps = []
            walks.validation_call(pipe, *inputs[call - 1], steps=3, callback=lambda i, t, x: steps.append(x.clone()))
            torch.cuda.synchronize()
            runs[graph] = steps
            engines |= {id(e) for _, e in pipe.unet._engines.values()}
            if graph:
                graphs |= {id(e.graph) for _, e in pipe.unet._engines.values()}
        assert len(runs[True]) == len(runs[False]) == 3
        for i, (a, b) in enumerate(zip(runs[True], runs[False])):
            assert torch.isfinite(b).all(), f'call {call} step {i + 1}: eager latents not finite'
            assert_bits_equal(a, b, f'call {call} step {i + 1}: latents')
    assert len(engines) == 1 and len(graphs) == 1, 'the second call must replay the engine\'s first captured graph'
