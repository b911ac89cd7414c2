"""Every MulPir response call goes through one pipeline: the single-client calls and a group of one client in the
many-clients call run the same kernels, device entry points only enqueue on the caller's stream, and the host
single-client call replays a captured graph."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import hecuda
from hecuda import pir
from oracle import oracle as orc
from test_gpu_pir_clients import GROUP, PIR_MODULI, Setup, contexts

SCANS = ("inner_product_plain_kernel", "inner_product_plain_small_kernel")  # the single-client first-dimension scans
CLIENT_SCANS = ("inner_product_plain_clients_kernel", "inner_product_plain_small_clients_kernel")
SHAPES = ("uint32 rows", "uint64 rows")


def setup(shape, indices_count):
    if shape == "uint32 rows":  # N = 4096 over the default PIR moduli (27 / 28 / 28 bits)
        n, t, entries, entry_size = 4096, 17, 3000, 1
        g, o = hecuda.Context(n, PIR_MODULI, t), orc.Context(n, PIR_MODULI, t)
    else:
        n, t, entries, entry_size = 64, 65537, 200, 24
        g, o = contexts(n, [55, 55, 55], t)
    return Setup(g, o, entries, entry_size, 2, indices_count, True, "hybridCompression", seed=n + indices_count)


def launches(names, kernels):
    """How many of `names` are launches of one of `kernels` (all are templates: the name ends in `<`)."""
    return sum(any(k + "<" in name for k in kernels) for name in names)


def device_response(s, client, indices_count, stream):
    """hecuda_mulpir_compute_response_device on `stream`; returns the output tensor (valid once the stream is done)."""
    import torch

    with torch.cuda.stream(stream):
        d_q = torch.from_numpy(client["query"].view(np.int64)).cuda()
        d_out = torch.empty((indices_count, s.server.chunkCount, 2, 1, s.o.n), dtype=torch.int64, device="cuda")
    stream.synchronize()
    dbs = s.server.databases
    handles = (C.c_void_p * len(dbs))(*[d._h for d in dbs])
    dims = (C.c_int32 * len(s.param.dimensions))(*s.param.dimensions)

    def call():
        hecuda._check(hecuda.load_library().hecuda_mulpir_compute_response_device(
            s.g._h, client["key"]._h, handles, len(dbs), dims, len(dims), s.server.chunkCount, d_q.data_ptr(),
            client["query"].shape[0], indices_count, d_out.data_ptr(), stream.cuda_stream))

    return call, d_out


def kernels(fn):
    """Names of the kernels `fn` runs, in the order they ran."""
    import torch
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    events = [e for e in prof.events() if e.device_type == DeviceType.CUDA and not e.name.startswith(("Memcpy", "Memset"))]
    return [e.name for e in sorted(events, key=lambda e: e.time_range.start)]


def test_device_calls_do_not_wait_for_the_callers_stream():
    import torch

    s = setup("uint64 rows", 1)
    client = s.client(10)
    want = s.server.computeResponse(client["query"], client["key"])
    stream = torch.cuda.Stream()
    respond, d_out = device_response(s, client, 1, stream)
    query, outputs = client["query"], s.param.expandedQueryCount
    expand_want = pir.PirUtil.expand(s.g, query, outputs, client["key"])
    with torch.cuda.stream(stream):
        d_q = torch.from_numpy(query.view(np.int64)).cuda()
        d_expanded = torch.empty((outputs,) + query.shape[1:], dtype=torch.int64, device="cuda")

    def expand():
        hecuda._check(hecuda.load_library().hecuda_mulpir_expand_device(
            s.g._h, client["key"]._h, d_q.data_ptr(), query.shape[0], outputs, d_expanded.data_ptr(), stream.cuda_stream))

    for call, out, expected in ((respond, d_out, want), (expand, d_expanded, expand_want)):
        call()  # the first call with this shape uploads its expansion plan
        stream.synchronize()
        with torch.cuda.stream(stream):
            out.zero_()
            torch.cuda._sleep(200_000_000)  # about 0.1 s of busy cycles ahead of the call
        call()
        assert not stream.query(), "the call waited for work queued on the caller's stream"
        stream.synchronize()
        assert np.array_equal(out.cpu().numpy().view(np.uint64), expected)
    s.close([client])
    s.g.close()


@pytest.mark.parametrize("indices_count", [1, 2])
@pytest.mark.parametrize("shape", SHAPES)
def test_a_group_of_one_runs_the_single_client_kernels(shape, indices_count):
    import torch

    s = setup(shape, indices_count)
    client = s.client(20, indices_count=indices_count)
    stream = torch.cuda.Stream()
    respond, d_out = device_response(s, client, indices_count, stream)

    def group_of_one():
        return s.server.computeResponses(client["query"][None], [client["key"]], indicesCount=indices_count)

    def single():
        respond()
        stream.synchronize()

    got = group_of_one()  # warm both calls
    single()
    assert np.array_equal(d_out.cpu().numpy().view(np.uint64), got[0])
    group_kernels, single_kernels = kernels(group_of_one), kernels(single)
    assert group_kernels == single_kernels
    assert launches(single_kernels, SCANS) == indices_count and launches(single_kernels, CLIENT_SCANS) == 0
    s.close([client])
    s.g.close()


@pytest.mark.parametrize("indices_count", [1, 2])
def test_the_last_lone_client_runs_the_single_client_scan(indices_count):
    s = setup("uint64 rows", indices_count)
    clients = [s.client(30 + c, indices_count=indices_count) for c in range(GROUP + 1)]
    queries = np.stack([c["query"] for c in clients])
    keys = [c["key"] for c in clients]
    got = s.server.computeResponses(queries, keys, indicesCount=indices_count)
    names = kernels(lambda: s.server.computeResponses(queries, keys, indicesCount=indices_count))
    assert launches(names, CLIENT_SCANS) == indices_count and launches(names, SCANS) == indices_count
    for j in (0, GROUP):
        assert np.array_equal(got[j], s.server.computeResponse(clients[j]["query"], keys[j], indicesCount=indices_count))
    s.close(clients)
    s.g.close()


def test_the_host_call_replays_a_captured_graph():
    import torch
    from torch.profiler import ProfilerActivity, profile

    s = setup("uint64 rows", 1)
    client = s.client(40)
    first = s.server.computeResponse(client["query"], client["key"])  # captures
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        second = s.server.computeResponse(client["query"], client["key"])
        torch.cuda.synchronize()
    runtime = [e.name for e in prof.events() if e.name.startswith("cuda")]
    assert any(name.startswith("cudaGraphLaunch") for name in runtime), runtime
    assert not any(name.startswith("cudaLaunchKernel") for name in runtime), runtime
    assert np.array_equal(first, second)
    s.close([client])
    s.g.close()
