"""``last_launch_count()`` against the kernels a call actually issues.  Each call of lg_forward, lg_assign and
lg_attention is repeated once under CUDA graph capture with nothing else in the capture, and the count the library
reports must equal the number of kernel nodes in the captured graph."""
import ctypes

import pytest
import torch

from lightglue_b200 import LightGlue, _cabi, synth

pytestmark = pytest.mark.gpu

PRECISIONS = ["fp32", "bf16", "bf16x3"]
CU_GRAPH_NODE_TYPE_KERNEL = 0


def kernel_nodes(graph):
    cu = ctypes.CDLL("libcuda.so.1")
    g, n = ctypes.c_void_p(graph.raw_cuda_graph()), ctypes.c_size_t(0)
    assert cu.cuGraphGetNodes(g, None, ctypes.byref(n)) == 0
    nodes = (ctypes.c_void_p * n.value)()
    assert cu.cuGraphGetNodes(g, nodes, ctypes.byref(n)) == 0
    kinds = [ctypes.c_int(-1) for _ in range(n.value)]
    for node, kind in zip(nodes, kinds):
        assert cu.cuGraphNodeGetType(ctypes.c_void_p(node), ctypes.byref(kind)) == 0
    return sum(k.value == CU_GRAPH_NODE_TYPE_KERNEL for k in kinds)


@pytest.fixture
def kernels(monkeypatch):
    """Wraps the library's kernel-running entry points; returns the list of kernel counts, one per call."""
    lib = _cabi.load()
    counts = []

    def counted(fn):
        def call(*args):
            rc = fn(*args)  # the call itself, which also does the one-time setup a capture must not
            if rc == 0:
                graph = torch.cuda.CUDAGraph(keep_graph=True)
                with torch.cuda.graph(graph):  # the same call again on the capturing stream (the last argument)
                    assert fn(*args[:-1], torch.cuda.current_stream().cuda_stream) == 0
                counts.append(kernel_nodes(graph))
            return rc
        return call

    for name in ("lg_forward", "lg_assign", "lg_attention"):
        monkeypatch.setattr(lib, name, counted(getattr(lib, name)))
    return counts


def matcher(precision, adaptive=False, input_dim=256):
    m = LightGlue(features=None, input_dim=input_dim, precision=precision, depth_confidence=0.95 if adaptive else -1,
                  width_confidence=0.99 if adaptive else -1)
    m.load_state_dict(synth.make_state_dict(input_dim=input_dim, adaptive=adaptive), strict=False)
    m.pruning_keypoint_thresholds = dict(LightGlue.pruning_keypoint_thresholds, flash=-1)  # prune at any size
    return m.eval().cuda()


def to_cuda(data):
    return {k: {kk: vv.cuda() for kk, vv in v.items()} for k, v in data.items()}


def check(m, kernels):
    assert len(kernels) == 1 and kernels[0] > 0, kernels
    assert m.last_launch_count() == kernels[0]


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("adaptive,input_dim", [(False, 256), (True, 256), (False, 128)])
def test_forward(precision, adaptive, input_dim, kernels):
    m = matcher(precision, adaptive, input_dim)
    data, _ = synth.make_pair(512, d=input_dim, seed=21)
    m(to_cuda(data))
    check(m, kernels)


@pytest.mark.parametrize("precision", PRECISIONS)
def test_forward_ragged(precision, kernels):
    m = matcher(precision)
    data, _ = synth.make_pair(400, b=2, seed=22)
    data["image0"]["num_keypoints"] = torch.tensor([400, 150])
    data["image1"]["num_keypoints"] = torch.tensor([260, 400])
    m(to_cuda(data))
    check(m, kernels)


@pytest.mark.parametrize("precision", PRECISIONS)
def test_forward_empty_side(precision, kernels):
    m = matcher(precision)
    data, _ = synth.make_pair(300, m=0, seed=23)
    m(to_cuda(data))
    check(m, kernels)
    assert kernels == [1]


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("M,N", [(200, 333), (100, 90)])  # Lp 384: tensor-core sweeps; Lp 128: CUDA-core sweeps
def test_assign(precision, M, N, kernels):
    m = matcher(precision)
    g = torch.Generator().manual_seed(M + N)
    x0, x1 = torch.randn(2, M, 256, generator=g), torch.randn(2, N, 256, generator=g)
    m.log_assignment_matrix(4, x0.cuda(), x1.cuda())
    check(m, kernels)


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("cross", [False, True])
def test_attention(precision, cross, kernels):
    m = matcher(precision)
    g = torch.Generator().manual_seed(24)
    q0, k0, v0 = (torch.randn(2, 4, 300, 64, generator=g).cuda() for _ in range(3))
    q1, k1, v1 = (torch.randn(2, 4, 517, 64, generator=g).cuda() for _ in range(3))
    m.attention(q0, k0, v0, q1, k1, v1, cross=cross)
    check(m, kernels)
