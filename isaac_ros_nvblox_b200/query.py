"""Point queries of one or several mappers on the GPU, with nvblox_torch's names and output layouts
(nvblox_torch/mapper.py:311-460 query_layer / query_differentiable_layer, nvblox_torch/sdf_query.py EsdfQuery).

    query_type   output (n x S)                 one mapper                       several mappers
    TSDF         [distance, weight]             written where the voxel exists   min distance, weight at it; {100, 0} if none
    ESDF         [distance]                     signed distance - radius         minimum (nvb_query_esdf's rule)
    ESDF_GRAD    [grad_x, grad_y, grad_z, distance]
    OCCUPANCY    [log_odds]                     max(log-odds, logOdds(0))        maximum

`mappers` is one Mapper (the single-mapper rules) or a sequence of them (more than one: the multi-mapper rules; a sequence of
one is that mapper alone, as nvblox_torch's EsdfQuery does). Queries are float32 CUDA tensors, (n, 3) points or, for the
ESDF, (n, 4) spheres {x, y, z, radius} (an (n, 3) query has radius 0). Outputs that a query never writes keep the value they
are pre-filled with: zeros for TSDF and OCCUPANCY, 100 (the unknown distance) for ESDF and ESDF_GRAD, as _maybe_allocate
does. The query is enqueued on torch's current stream after the work already on it and on every mapper; no host
synchronisation.
"""
import ctypes as C
import enum

import torch

from ._lib import check
from .mapper import _device_points

ESDF_UNKNOWN_DISTANCE = 100.0  # nvblox_torch/sdf_query.cuh:30-31 (constants.esdf_unknown_distance())


class QueryType(enum.Enum):
    TSDF = 0
    ESDF = 1
    ESDF_GRAD = 2
    OCCUPANCY = 3


_WIDTH = {QueryType.TSDF: 2, QueryType.ESDF: 1, QueryType.ESDF_GRAD: 4, QueryType.OCCUPANCY: 1}
_FILL = {QueryType.TSDF: 0.0, QueryType.ESDF: ESDF_UNKNOWN_DISTANCE, QueryType.ESDF_GRAD: ESDF_UNKNOWN_DISTANCE,
         QueryType.OCCUPANCY: 0.0}


def _mapper_list(mappers):
    ms = list(mappers) if isinstance(mappers, (list, tuple)) else [mappers]
    if not ms:
        raise ValueError("no mappers to query")
    dev = ms[0]._device
    if any(m._device != dev for m in ms):
        raise ValueError("the mappers of one query must be on the same device")
    return ms, dev


def _run(ms, query_type, query, output):
    dev = ms[0]._device
    esdf = query_type in (QueryType.ESDF, QueryType.ESDF_GRAD)
    q = _device_points(query, (3, 4) if esdf else 3, dev, "query")
    n = q.shape[0]
    if esdf and q.shape[1] == 3:
        q = torch.cat([q, torch.zeros((n, 1), dtype=q.dtype, device=q.device)], dim=1)
    width = _WIDTH[query_type]
    if output is None:
        output = torch.full((n, width), _FILL[query_type], dtype=torch.float32, device=q.device)
    else:
        _device_points(output, width, dev, "output")
        if output.shape[0] != n or not output.is_contiguous():
            raise ValueError("output must be a contiguous (%d, %d) tensor" % (n, width))
    handles = (C.c_void_p * len(ms))(*[m._h.value for m in ms])
    stream = C.c_void_p(torch.cuda.current_stream(q.device).cuda_stream)
    L = ms[0]._L
    if esdf:
        rc = L.nvb_query_esdf(handles, len(ms), q.data_ptr(), n, 1 if query_type == QueryType.ESDF_GRAD else 0,
                              output.data_ptr(), stream)
    elif query_type == QueryType.TSDF:
        rc = L.nvb_query_tsdf(handles, len(ms), q.data_ptr(), n, output.data_ptr(), stream)
    else:
        rc = L.nvb_query_occupancy(handles, len(ms), q.data_ptr(), n, output.data_ptr(), stream)
    check(rc)
    return output


def query_layer(mappers, query_type, query, output=None):
    """Mapper.query_layer (nvblox_torch/mapper.py:326-412): the (n, S) tensor of the table above, `output` if given."""
    ms, _ = _mapper_list(mappers)
    return _run(ms, QueryType(query_type), query, output)


class EsdfQuery(torch.autograd.Function):
    """EsdfQuery (nvblox_torch/sdf_query.py:16-110): the signed distance of each sphere to the surface, differentiable with
    respect to the query. backward returns grad_out * [gx, gy, gz, -1] (the radius column only for (n, 4) spheres)."""

    @staticmethod
    def forward(ctx, query_spheres, mappers, out_tensor=None):
        ms, _ = _mapper_list(mappers)
        xyzd = _run(ms, QueryType.ESDF_GRAD, query_spheres, out_tensor)
        ctx.cols = query_spheres.shape[1]
        ctx.save_for_backward(xyzd)
        return xyzd[:, 3].clone()

    @staticmethod
    def backward(ctx, grad_output):
        grad = None
        if ctx.needs_input_grad[0]:
            (xyzd,) = ctx.saved_tensors
            d = xyzd.clone()
            d[:, 3] = -1.0
            grad = (grad_output.unsqueeze(-1) * d)[:, :ctx.cols]
        return grad, None, None


def query_differentiable_layer(mappers, query_type, query, output=None):
    """Mapper.query_differentiable_layer (nvblox_torch/mapper.py:414-459): ESDF only, an (n,) tensor that supports autograd."""
    if QueryType(query_type) != QueryType.ESDF:
        raise NotImplementedError("only the ESDF layer has a differentiable query")
    return EsdfQuery.apply(query, mappers, output)
