"""Test harness: ranks as THREADS of one process for the host simulation of the kernel sources -- a stand-in for the calls
``parcels_b200.distributed`` makes on ``torch.distributed`` (all_reduce over a thread barrier) and a lock that serialises the engine
calls of the ranks (the simulated device runs a kernel as a loop over global thread / block indices and its atomics are plain host
operations).  Used by scripts/decomposed_threads_check.py and scripts/fuzz_hostsim_r2.py."""
import threading

import torch


class ThreadGroup:
    """all_reduce over the threads of one process (what run_decomposed_p2p / execute_decomposed ask of torch.distributed)."""

    class ReduceOp:
        SUM, MIN, MAX = "sum", "min", "max"

    def __init__(self, world):
        self.world = world
        self.barrier = threading.Barrier(world)
        self.slots = [None] * world

    def member(self, rank):
        group = self

        class Member:
            ReduceOp = ThreadGroup.ReduceOp

            @staticmethod
            def get_rank():
                return rank

            @staticmethod
            def get_world_size():
                return group.world

            @staticmethod
            def get_backend():
                return "threads"

            @staticmethod
            def all_reduce(t, op="sum"):
                group.slots[rank] = t.clone()
                group.barrier.wait()
                stack = torch.stack(group.slots)
                res = stack.sum(0) if op == "sum" else (stack.min(0).values if op == "min" else stack.max(0).values)
                group.barrier.wait()  # everybody has read the slots before the next collective overwrites them
                t.copy_(res)

            @staticmethod
            def all_gather_into_tensor(out, t):
                group.slots[rank] = t.clone()
                group.barrier.wait()
                res = torch.cat(group.slots)
                group.barrier.wait()
                out.copy_(res)

            @staticmethod
            def all_gather_object(out, obj):
                group.slots[rank] = obj
                group.barrier.wait()
                out[:] = list(group.slots)
                group.barrier.wait()

        return Member


_serialised = False


def serialise_engine_calls():
    """Wrap every Engine method in one process-wide lock (idempotent)."""
    global _serialised
    if _serialised:
        return
    from parcels_b200.engine import Engine

    device_lock = threading.RLock()

    def locked(method):
        def call(*args, **kw):
            with device_lock:
                return method(*args, **kw)

        return call

    for name, method in list(vars(Engine).items()):
        if callable(method) and not name.startswith("__") and not isinstance(method, (staticmethod, classmethod)):
            setattr(Engine, name, locked(method))
    _serialised = True


def run_ranks(world, rank_main):
    """rank_main(rank, dist) on ``world`` threads; returns the list of results, re-raises the first exception of any rank."""
    group = ThreadGroup(world)
    results, errors = [None] * world, []

    def body(r):
        try:
            results[r] = rank_main(r, group.member(r))
        except BaseException as e:  # noqa: BLE001 -- a dead rank would leave the others in the barrier
            errors.append(e)
            group.barrier.abort()

    threads = [threading.Thread(target=body, args=(r,)) for r in range(world)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    if errors:
        first = [e for e in errors if not isinstance(e, threading.BrokenBarrierError)]
        raise (first or errors)[0]
    return results
