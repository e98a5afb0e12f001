"""
Communicator shim: the handful of mpi4py-style members the FFTPower path touches
(`rank`, `size`, `allreduce`, `allgather`, `bcast`, `alltoall`, `barrier`; SURVEY.md §2.3), over
`torch.distributed` (NCCL on GPUs, gloo in CPU tests).  One process per GPU.

Small Python objects travel with the *_object collectives; tensors (particle columns, packed FFT
blocks, histograms) use all_to_all_single / all_reduce directly on device memory.
"""
import os

import numpy
import torch


class SelfComm(object):
    """single-process communicator (no torch.distributed needed)"""
    rank = 0
    size = 1

    def allreduce(self, x, op="sum"):
        return x

    def allgather(self, x):
        return [x]

    def bcast(self, x, root=0):
        return x

    def alltoall(self, xs):
        return list(xs)

    def barrier(self):
        pass

    Barrier = barrier

    # tensor collectives
    def allreduce_tensor(self, t, op="sum"):
        return t

    def all_to_all_single(self, out, inp, out_splits=None, in_splits=None):
        out.copy_(inp)
        return out

    def alltoall_ints(self, xs):
        return [int(x) for x in xs]

    def allreduce_floats(self, xs):
        return [float(x) for x in xs]

    def __repr__(self):
        return "SelfComm()"


class TorchComm(object):
    """wraps a torch.distributed process group"""

    def __init__(self, group=None):
        import torch.distributed as dist
        if not dist.is_initialized():
            raise RuntimeError("torch.distributed is not initialized")
        self._dist = dist
        self.group = group
        self.rank = dist.get_rank(group)
        self.size = dist.get_world_size(group)
        self._backend = dist.get_backend(group)

    _OPS = None

    def _op(self, op):
        R = self._dist.ReduceOp
        return {"sum": R.SUM, "min": R.MIN, "max": R.MAX, "lor": R.MAX}[op if isinstance(op, str) else "sum"]

    def _device(self):
        if self._backend == "nccl":
            return torch.device("cuda", torch.cuda.current_device())
        return torch.device("cpu")

    # ---- python-object collectives (scalars, small arrays, dicts)
    def allreduce(self, x, op="sum"):
        if isinstance(x, torch.Tensor):
            return self.allreduce_tensor(x.clone(), op)
        a = numpy.asarray(x)
        if a.dtype == bool:
            a = a.astype("i8")
        t = torch.from_numpy(numpy.ascontiguousarray(a).reshape(-1).copy()).to(self._device())
        self._dist.all_reduce(t, op=self._op(op), group=self.group)
        r = t.cpu().numpy().reshape(a.shape)
        if numpy.ndim(x) == 0 and not isinstance(x, numpy.ndarray):
            r = r.reshape(()).item()
            if isinstance(x, (bool, numpy.bool_)):
                r = bool(r)
        return r

    def allgather(self, x):
        out = [None] * self.size
        self._dist.all_gather_object(out, x, group=self.group)
        return out

    def bcast(self, x, root=0):
        box = [x]
        self._dist.broadcast_object_list(box, src=root, group=self.group)
        return box[0]

    def alltoall(self, xs):
        gathered = self.allgather(list(xs))
        return [gathered[src][self.rank] for src in range(self.size)]

    def barrier(self):
        self._dist.barrier(group=self.group)

    Barrier = barrier

    # ---- tensor collectives (device memory)
    def allreduce_tensor(self, t, op="sum"):
        if self._backend == "gloo" and t.is_cuda:
            # gloo reduces host memory: several ranks sharing one GPU (tests) go through a host copy
            h = t.cpu()
            self._dist.all_reduce(h, op=self._op(op), group=self.group)
            t.copy_(h)
            return t
        self._dist.all_reduce(t, op=self._op(op), group=self.group)
        return t

    def all_to_all_single(self, out, inp, out_splits=None, in_splits=None):
        if self._backend == "gloo":
            # gloo has no all_to_all_single: emulate with all_to_all on chunk lists
            n = self.size
            ins = list(inp.split(in_splits if in_splits is not None else inp.shape[0] // n))
            outs = list(out.split(out_splits if out_splits is not None else out.shape[0] // n))
            ins = [c.contiguous() for c in ins]
            outs_c = [torch.empty_like(c) for c in outs]
            self._gloo_all_to_all(outs_c, ins)
            for o, c in zip(outs, outs_c):
                o.copy_(c)
            return out
        self._dist.all_to_all_single(out, inp, out_splits, in_splits, group=self.group)
        return out

    def alltoall_ints(self, xs):
        """alltoall of one integer per destination, as ONE small tensor collective (no pickling)"""
        dev = self._device()
        inp = torch.tensor([int(x) for x in xs], dtype=torch.int64, device=dev)
        out = torch.empty_like(inp)
        self.all_to_all_single(out, inp)
        return [int(v) for v in out.cpu().tolist()]

    def allreduce_floats(self, xs):
        """sum-allreduce of a few scalars in one collective"""
        t = torch.tensor([float(x) for x in xs], dtype=torch.float64, device=self._device())
        self._dist.all_reduce(t, group=self.group)
        return [float(v) for v in t.cpu().tolist()]

    def _gloo_all_to_all(self, outs, ins):
        if any(t.is_cuda for t in outs + ins):
            # gloo sends host memory: stage device chunks through host copies
            h_outs = [o.cpu() for o in outs]
            self._gloo_all_to_all(h_outs, [c.cpu() for c in ins])
            for o, h in zip(outs, h_outs):
                o.copy_(h)
            return
        reqs = []
        for peer in range(self.size):
            if peer == self.rank:
                outs[peer].copy_(ins[peer])
                continue
            reqs.append(self._dist.isend(ins[peer], dst=peer, group=self.group))
            reqs.append(self._dist.irecv(outs[peer], src=peer, group=self.group))
        for r in reqs:
            r.wait()

    def __repr__(self):
        return "TorchComm(rank=%d, size=%d, backend=%s)" % (self.rank, self.size, self._backend)


_world = None


def world():
    """COMM_WORLD equivalent: the default torch.distributed group when initialised (or when
    launched under torchrun, in which case it is initialised here), else a SelfComm"""
    global _world
    import torch.distributed as dist
    if _world is not None:
        if isinstance(_world, SelfComm) and dist.is_available() and dist.is_initialized():
            _world = TorchComm()
        return _world
    if dist.is_available() and dist.is_initialized():
        _world = TorchComm()
    elif dist.is_available() and "RANK" in os.environ and "WORLD_SIZE" in os.environ \
            and int(os.environ["WORLD_SIZE"]) > 1:
        backend = "nccl" if torch.cuda.is_available() else "gloo"
        if backend == "nccl":
            torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", 0)))
        dist.init_process_group(backend=backend)
        _world = TorchComm()
    else:
        _world = SelfComm()
    return _world
