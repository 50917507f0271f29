"""Multi-GPU plumbing: one process per GPU, utterances sharded by batch (SURVEY 8e).

Exactly two collectives, as the north star prescribes: one broadcast of the packed weight arena
from rank 0 at start-up and a gather of the output waveforms to rank 0 per step.  Shard sizes are
static for a job, so they are exchanged ONCE when a `WaveformGather` is built (start-up, like the
weight broadcast) and never in the step.  The functions take the process group's backend as given,
so the same code runs under NCCL on the GPUs and under gloo on CPU tensors in the tests (world_size 2).

`run_on_devices` is the other form, with no process group: the caller spawns one worker process per extra device and
each runs a shard of independent jobs (VoiceFixer.restore_files(..., gpus=N)), reporting only its outcome back."""
import os
import torch
import torch.distributed as dist


def init_from_env(backend=None):
    """Initialises torch.distributed from torchrun's environment; returns (rank, world, local_rank)."""
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    if world > 1 and not dist.is_initialized():
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        os.environ.setdefault("MASTER_PORT", "29500")
        if backend is None:
            backend = "nccl" if torch.cuda.is_available() else "gloo"
        kw = {}
        if backend == "nccl":
            kw["device_id"] = torch.device(f"cuda:{local}")
        dist.init_process_group(backend=backend, rank=rank, world_size=world, **kw)
    return rank, world, local


def shard_range(n_items, rank, world):
    """Contiguous shard [lo, hi) of n_items for `rank`; the first n_items % world ranks get one extra."""
    base, rem = divmod(n_items, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def broadcast_arena(table, arena, device, src=0):
    """Rank `src` holds (table, arena uint8 tensor); everyone returns (table, arena on `device`).
    One broadcast of the layout (python object) and one of the bytes (NCCL over NVLink on GPUs)."""
    if not dist.is_initialized() or dist.get_world_size() == 1:
        return table, arena
    meta = [table, int(arena.numel()) if arena is not None else 0]
    dist.broadcast_object_list(meta, src=src)
    table, nbytes = meta
    if dist.get_rank() != src:
        arena = torch.empty(nbytes, dtype=torch.uint8, device=device)
    dist.broadcast(arena, src=src)
    return table, arena


class WaveformGather:
    """The per-step collective: local_out (b_r, L) on each rank -> (sum b_r, L) on rank dst.

    Built once per job: the shard sizes are exchanged here (one all_gather of a single integer at start-up) and the
    receive buffers on rank dst are allocated once, so `__call__` issues exactly ONE collective (dist.gather) and no host
    synchronisation.  Ragged shards are padded to the largest shard inside the send buffer."""

    def __init__(self, n_local, length, dtype, device, dst=0):
        self.dst, self.n_local, self.length = dst, int(n_local), int(length)
        self.active = dist.is_initialized() and dist.get_world_size() > 1
        self.sizes = [self.n_local]
        self.recv = self.out = self.send = None
        if not self.active:
            return
        world, self.rank = dist.get_world_size(), dist.get_rank()
        sizes = [torch.zeros(1, dtype=torch.int64, device=device) for _ in range(world)]
        dist.all_gather(sizes, torch.tensor([self.n_local], dtype=torch.int64, device=device))
        self.sizes = [int(s.item()) for s in sizes]                   # start-up only
        self.bmax = max(self.sizes)
        if self.n_local != self.bmax:
            self.send = torch.zeros(self.bmax, self.length, dtype=dtype, device=device)
        if self.rank == dst:
            # one contiguous (world, bmax, L) buffer: with equal shards the gathered result is a view of it, no copy
            self.out = torch.empty(world, self.bmax, self.length, dtype=dtype, device=device)
            self.recv = [self.out[r] for r in range(world)]

    @property
    def total_items(self):
        return sum(self.sizes)

    def __call__(self, local_out):
        """One dist.gather on the current stream; returns the gathered (sum b_r, L) tensor on rank dst, None elsewhere."""
        if not self.active:
            return local_out
        src = local_out
        if self.send is not None:
            self.send[: self.n_local].copy_(local_out)
            src = self.send
        dist.gather(src.contiguous(), self.recv, dst=self.dst)
        if self.rank != self.dst:
            return None
        if all(n == self.bmax for n in self.sizes):
            return self.out.view(-1, self.length)
        return torch.cat([self.out[r, :n] for r, n in enumerate(self.sizes)], 0)


def gather_waveforms(local_out, dst=0):
    """One-shot convenience form (builds a WaveformGather for this call: the size exchange is then part of it)."""
    return WaveformGather(local_out.shape[0], local_out.shape[1], local_out.dtype, local_out.device, dst)(local_out)


def _outcome(target, device, shard, args):
    """target's outcome on one shard: None when it is done, else (input index, exception type, message, exception).
    target returns None or (the input index it failed on, the exception); an exception it raises itself counts as a
    failure at the shard's first input."""
    try:
        failed = target(device, shard, args)
    except Exception as e:                               # noqa: BLE001 - reported to the caller
        failed = (shard[0], e)
    if failed is None:
        return None
    index, e = failed
    return int(index), type(e), str(e), e


def _worker(target, device, shard, args, conn):
    """A worker process's body: runs its shard and sends the outcome, without the exception object, to the caller."""
    outcome = _outcome(target, device, shard, args)
    if outcome is not None:
        outcome = outcome[:3]
    try:
        conn.send(outcome)
    except Exception:                                    # noqa: BLE001 - an exception type that does not pickle
        index, etype, message = outcome
        conn.send((index, RuntimeError, f"{etype.__name__}: {message}"))
    conn.close()


def run_on_devices(shards, target, args):
    """Runs target(device, shard, args) for each (device, shard) of shards, one process per shard after the first,
    started with the spawn method (CUDA cannot be forked), while the calling process runs the first shard itself.
    target must be a module-level function (the workers import it) and returns None when its shard is done or
    (failing input index, exception) for the first input it failed on.

    Returns once every shard has finished; every process is joined before this returns or raises, and terminated
    first if the caller is interrupted.  Then, if any shard failed, raises the failure with the lowest input index: the
    exception itself for the caller's shard, a new one of the same type and message for a worker's (RuntimeError
    "<type>: <message>" for a type that cannot be rebuilt from its message).  A worker that exits without reporting
    raises RuntimeError naming its device and exit code."""
    import multiprocessing
    from multiprocessing.connection import wait
    ctx = multiprocessing.get_context("spawn")
    procs = []
    try:
        for device, shard in shards[1:]:
            recv, send = ctx.Pipe(duplex=False)
            p = ctx.Process(target=_worker, args=(target, device, shard, args, send), daemon=True,
                            name=f"vfx-device-{device}")
            p.start()
            send.close()
            procs.append((device, p, recv))
        outcomes = [_outcome(target, shards[0][0], shards[0][1], args)] if shards else []
        for (device, p, recv), (_, shard) in zip(procs, shards[1:]):
            wait([recv, p.sentinel])
            try:
                reported, outcome = recv.poll(), None
                if reported:
                    outcome = recv.recv()
            except EOFError:                             # it died while sending
                reported = False
            p.join()
            if not reported:
                outcome = (shard[0], RuntimeError,
                           f"the worker process of device {device} exited with code {p.exitcode} without reporting")
            outcomes.append(outcome)
    finally:
        for _, p, recv in procs:
            if p.is_alive():
                p.terminate()
            p.join()
            recv.close()
    failed = [o for o in outcomes if o is not None]
    if not failed:
        return
    first = min(failed, key=lambda o: o[0])
    if len(first) == 4:
        raise first[3]
    _, etype, message = first
    try:
        e = etype(message)
    except Exception:                                    # noqa: BLE001
        e = RuntimeError(f"{etype.__name__}: {message}")
    raise e
