"""One forward layer loop and one step-graph build (CPU, with the torch stand-ins of the kernels).

The inference forward and the training forward enqueue the same stage calls with the same flags, apart from the
accumulator clears that only the inference path asks for.  The backward of `differentiable_rollout` recomputes every
step's graph and forward with the calls, flags and inputs its forward used, in radius, fixed-graph and cutoff modes."""
import pytest
import torch

from distegnn_b200 import _lib, differentiable_rollout, synth
from distegnn_b200.shards import CSRGraph
from tests.shadow_backend import ShadowBackend
from tests.test_cutoff import CutoffStandIn
from tests.test_rollout import _cpu_case
from tests.test_rollout_grad import RolloutGradStandIn

GRAPH = ("radius_graph_into", "edge_lengths", "cutoff_into")
FORWARD = GRAPH + ("embed", "edge_layer", "virtual_layer", "node_layer", "virtual_update")
ZERO = _lib.FLAG_ZERO_AGG | _lib.FLAG_ZERO_VSUM
POS_ARG = dict(radius_graph_into=1, edge_lengths=2, cutoff_into=2, embed=2)   # the positions each call reads


def recording(be):
    """Wrap every stage method of `be`: be.trace gets (name, flags or None, which arguments are None, the positions read
    by a graph build or the embedding, as a copy)."""
    be.trace = []
    for name in FORWARD + ("rollout_advance", "rollout_advance_bwd"):
        fn = getattr(be, name, None)
        if fn is None:
            continue

        def call(*a, _fn=fn, _name=name, **k):
            if _name == "radius_graph_into" and a[0].capacity == 0:    # the count-only probe of the first capacity
                return _fn(*a, **k)
            flags = a[1] if isinstance(a[1], int) else None
            pos = a[POS_ARG[_name]].clone() if _name in POS_ARG else None
            be.trace.append((_name, flags, tuple(x is None for x in a), pos))
            return _fn(*a, **k)
        setattr(be, name, call)
    return be


def test_inference_and_training_forward_enqueue_the_same_stages():
    m = _cpu_case(n=120)[0]
    inp = synth.make_partitions(synth.WORKLOADS["fluid113k"], n_nodes=120, seed=0)[0]
    m._backend = be = recording(ShadowBackend())
    with torch.no_grad():
        m(**inp)
    infer = be.trace
    be.trace = []
    out, X = m(**inp)
    assert out.requires_grad and X.requires_grad
    train = be.trace
    L = m.n_layers
    assert len(infer) == len(train) == 2 + 4 * L
    assert [(c[0], c[1] if c[1] is None else c[1] & ~ZERO) for c in infer] == \
        [(c[0], c[1]) for c in train]
    # only the inference path clears the accumulators; both read loc_mean and hv0 through the INIT update's pointers
    assert all(c[1] & ZERO for c in infer if c[0] in ("node_layer", "virtual_update"))
    assert not any(c[1] & ZERO for c in train if c[1] is not None)
    init_i, init_t = infer[1], train[1]
    assert init_i[0] == init_t[0] == "virtual_update" and init_i[1] & _lib.FLAG_INIT
    assert init_i[2][8:10] == init_t[2][8:10] == (False, False)


def _steps(trace, split):
    """The forward-family calls of each step: the segments of `trace` that end at a call named `split`."""
    segs, cur = [], []
    for c in trace:
        if c[0] == split:
            segs.append(cur)
            cur = []
        elif c[0] in FORWARD:
            cur.append(c)
    return segs


def _nbody_graph(node):
    N = node["node_loc"].shape[0]
    i, j = torch.meshgrid(torch.arange(N), torch.arange(N), indexing="ij")
    keep = (i != j) & (node["data_batch"][i] == node["data_batch"][j]) & ((i + j) % 3 == 0)
    return CSRGraph.from_edge_index(torch.stack([i[keep], j[keep]]), N)[0]


@pytest.mark.parametrize("mode", ["radius", "fixed", "cutoff_radius", "cutoff_fixed"])
def test_differentiable_rollout_backward_recomputes_the_forward_steps(mode):
    m, node, r, _ = _cpu_case(n=120)
    steps = 3
    kw = dict(radius=r) if mode.endswith("radius") else dict(graph=_nbody_graph(node))
    if mode.startswith("cutoff"):
        kw["cutoff_rate"] = 0.5
    m._backend = be = recording(CutoffStandIn() if mode.startswith("cutoff") else RolloutGradStandIn())
    leaf = {k: (v.clone().requires_grad_(True) if v.is_floating_point() else v) for k, v in node.items()}
    res = differentiable_rollout(m, **leaf, steps=steps, speed_col=0, **kw)
    fwd = _steps(be.trace, "rollout_advance")
    be.trace = []
    (res.trajectory.sum() + res.virtual_locs.sum()).backward()
    res.check()
    bwd = _steps(be.trace, "rollout_advance_bwd")[::-1]
    assert len(fwd) == len(bwd) == steps
    graph_calls = {"radius": ["radius_graph_into"], "fixed": ["edge_lengths"],
                   "cutoff_radius": ["radius_graph_into", "cutoff_into"], "cutoff_fixed": ["cutoff_into"]}[mode]
    for t, (f, b) in enumerate(zip(fwd, bwd)):
        assert [c[0] for c in f] == [c[0] for c in b] == graph_calls + ["embed", "virtual_update"] + \
            ["edge_layer", "virtual_layer", "node_layer", "virtual_update"] * m.n_layers, t
        assert [c[1] if c[1] is None else c[1] & ~ZERO for c in f] == [c[1] for c in b], t
        for cf, cb in zip(f, b):
            if cf[0] in GRAPH:                                 # the same build, from the same positions
                assert cf[2] == cb[2], (t, cf[0])
            if cf[3] is not None:
                assert torch.equal(cf[3], cb[3]), (t, cf[0])
        assert b[len(graph_calls) + 1][1] & _lib.FLAG_INIT_CENTROID == (_lib.FLAG_INIT_CENTROID if t else 0)
