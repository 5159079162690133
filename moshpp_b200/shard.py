"""Sequence sharding over the GPUs of one box (SURVEY.md 8(e), BASELINE config 5).

Sequences are independent (nothing is shared but the static model), so the path shards with no data-path
collective: rank 0 owns the observations of every sequence, scatters each one to the rank that will solve it,
every rank solves its sequences on its own GPU, and the per-frame result rows travel back to rank 0.  The scatter
and the gather are grouped point-to-point transfers of ``torch.distributed`` (NCCL over NVLink on GPUs, gloo in the
CPU tests); on GPUs the received tensors never touch the host: the C-ABI takes and returns device pointers
(``mosh2_job_upload_device`` / ``mosh2_job_download_device``).  One process per GPU; launch with torchrun.
"""
from __future__ import annotations

from typing import Callable, Dict, List, Optional, Sequence

import numpy as np


def assign_sequences(frame_counts: Sequence[int], world_size: int) -> List[List[int]]:
    """Longest-processing-time-first assignment of sequences to ranks (balanced by frame count)."""
    order = sorted(range(len(frame_counts)), key=lambda i: (-frame_counts[i], i))
    load = [0] * world_size
    out: List[List[int]] = [[] for _ in range(world_size)]
    for i in order:
        r = min(range(world_size), key=lambda k: (load[k], k))
        out[r].append(i)
        load[r] += frame_counts[i]
    for r in range(world_size):
        out[r].sort()
    return out


def _device(dist):
    import torch
    if dist.get_backend() == 'nccl':
        return torch.device('cuda', torch.cuda.current_device())
    return torch.device('cpu')


def _run_p2p(ops):
    import torch.distributed as dist
    if ops:
        for q in dist.batch_isend_irecv(ops):
            q.wait()


def scatter_observations(obs_list, vis_list, assignment: List[List[int]], shapes: List[tuple], src: int = 0):
    """Rank ``src`` holds every sequence's observations (``obs_list[i]``: F x M x 3 float32 tensor or array, host or
    device; ``vis_list[i]``: F x M uint8); every rank gets {seq: (obs, vis)} tensors on its own device for the
    sequences assigned to it.  ``shapes[i] = (F_i, M_i)`` is known on every rank (it is derived from the job list).
    All transfers go out as one grouped batch."""
    import torch
    import torch.distributed as dist
    rank, world = dist.get_rank(), dist.get_world_size()
    dev = _device(dist)

    def on_dev(a, dtype):
        t = a if isinstance(a, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(a))
        return t.to(device=dev, dtype=dtype, non_blocking=True).contiguous()

    mine: Dict[int, tuple] = {}
    ops, keep = [], []
    if rank == src:
        for r in range(world):
            for i in assignment[r]:
                o, v = on_dev(obs_list[i], torch.float32), on_dev(vis_list[i], torch.uint8)
                if r == src:
                    mine[i] = (o, v)
                else:
                    keep += [o, v]
                    ops += [dist.P2POp(dist.isend, o, r), dist.P2POp(dist.isend, v, r)]
    else:
        for i in assignment[rank]:
            F, M = shapes[i]
            o = torch.empty((F, M, 3), dtype=torch.float32, device=dev)
            v = torch.empty((F, M), dtype=torch.uint8, device=dev)
            mine[i] = (o, v)
            ops += [dist.P2POp(dist.irecv, o, src), dist.P2POp(dist.irecv, v, src)]
    _run_p2p(ops)
    return mine


def gather_results(local: Dict[int, 'object'], assignment: List[List[int]], row_widths: List[int], shapes: List[tuple],
                   dst: int = 0):
    """Gathers per-sequence result rows (one float32 tensor F_i x row_widths[i] per sequence on the rank's device) to
    rank ``dst``.  Returns {seq: tensor on dst's device} on dst, {} elsewhere."""
    import torch
    import torch.distributed as dist
    rank, world = dist.get_rank(), dist.get_world_size()
    dev = _device(dist)
    out: Dict[int, 'torch.Tensor'] = {}
    ops = []
    if rank == dst:
        for r in range(world):
            for i in assignment[r]:
                if r == dst:
                    out[i] = local[i]
                else:
                    out[i] = torch.empty((shapes[i][0], row_widths[i]), dtype=torch.float32, device=dev)
                    ops.append(dist.P2POp(dist.irecv, out[i], r))
    else:
        for i in assignment[rank]:
            ops.append(dist.P2POp(dist.isend, local[i].contiguous(), dst))
    _run_p2p(ops)
    return out


def solve_sharded(frame_counts: Sequence[int], n_markers: Sequence[int], row_widths: Sequence[int],
                  solve_fn: Callable[[Dict[int, tuple]], Dict[int, 'object']], obs_list=None, vis_list=None):
    """Scatter -> per-rank solves -> gather.  ``solve_fn({seq: (obs, vis)})`` gets this rank's sequences as tensors on
    the rank's device and returns {seq: F x width float32 tensor on the same device}.  Returns
    ({seq: rows} on rank 0 / {} elsewhere, assignment)."""
    import torch.distributed as dist
    world = dist.get_world_size()
    assignment = assign_sequences(list(frame_counts), world)
    shapes = [(int(f), int(m)) for f, m in zip(frame_counts, n_markers)]
    mine = scatter_observations(obs_list, vis_list, assignment, shapes)
    local = solve_fn(mine)
    return gather_results(local, assignment, list(row_widths), shapes), assignment


class GpuRankSolver:
    """This rank's share of a sharded run on its GPU.  Sequences that share a pack (one subject: body model, shape and
    marker layout, as in BASELINE config 5) are solved by ONE launch: a batch job holds them back to back on its frame
    axis, its chunks are planned for all of them together (chmosh.plan_chunk_len: whole waves of one chunk per SM) and
    never straddle a sequence.  Different subjects get a job each, on their own streams."""

    def __init__(self, packs: Dict[int, object], options, frame_counts: Dict[int, int], device: int, *,
                 chunk_warmup: int, warmup_full: int, sm_budget: Optional[int] = None, precision=None):
        from . import lib
        from .chmosh import NUM_SMS, first_chunk_extra, plan_chunk_len
        sm_budget = NUM_SMS if sm_budget is None else sm_budget
        self.device = device
        prec = lib.MOSH2_F32 if precision is None else precision
        extra = first_chunk_extra(chunk_warmup, warmup_full)
        common = plan_chunk_len(list(frame_counts.values()), sm_budget, chunk_warmup, warmup_full, first_extra=extra)
        groups: Dict[int, List[int]] = {}
        for i in frame_counts:
            groups.setdefault(id(packs[i]), []).append(i)
        self.models, self.jobs, self.where = [], [], {}
        for ids in groups.values():
            model = lib.Model(packs[ids[0]], device=device)
            counts = [int(frame_counts[i]) for i in ids]
            job = model.job(counts, options, chunk_len=common if common < max(counts) else 0, chunk_warmup=chunk_warmup,
                            warmup_full=warmup_full, precision=prec, first_extra=extra)
            self.models.append(model)
            self.jobs.append(job)
            for k, i in enumerate(ids):
                self.where[i] = (job, int(job.seq_offsets[k]), counts[k])
        self.chunk_len = common
        self.reports = []
        self.row_width = self.jobs[0].row_width

    def __call__(self, mine: Dict[int, tuple]) -> Dict[int, 'object']:
        import torch
        stream = torch.cuda.current_stream().cuda_stream
        for i, (o, v) in mine.items():                 # device-to-device, ordered after the producer (NCCL) stream
            job, f0, n = self.where[i]
            job.upload_device_range(f0, n, o.data_ptr(), False, v.data_ptr(), stream)
        from .chmosh import BOUNDARY_TOL, launch_verified
        self.reports = [launch_verified(job, BOUNDARY_TOL['fast'])[1] for job in self.jobs]   # launch + boundary check + repair
        torch.cuda.current_stream().synchronize()      # the row buffers below are written on the jobs' own streams
        out = {}
        for job in self.jobs:
            rows = torch.empty((job.n_frames, job.row_width), dtype=torch.float32, device=f'cuda:{self.device}')
            job.download_device(rows.data_ptr())       # packs on the job's stream and waits for it
            for i, (jb, f0, n) in self.where.items():
                if jb is job and i in mine:
                    out[i] = rows[f0:f0 + n]
        return out

    def span_ms(self) -> float:
        """Device time of the last solve: per job the sum over its launches (first launch over all chunks + repair
        launches, CUDA events on the job's stream); jobs of different subjects run concurrently on their own streams, so
        the rank's time is the maximum over its jobs."""
        return max(float(sum(r['kernel_ms'])) for r in self.reports)

    def num_chunks(self) -> int:
        return sum(j.num_chunks for j in self.jobs)

    def totals(self) -> Dict[str, int]:
        agg: Dict[str, int] = {}
        for j in self.jobs:
            for k, v in j.totals().items():
                agg[k] = agg.get(k, 0) + v
        return agg

    def close(self):
        for j in self.jobs:
            j.close()
        for m in self.models:
            m.close()
