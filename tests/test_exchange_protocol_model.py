"""Model check of the bitmask-exchange protocol (DESIGN.md section 5; lb200_ctx::Peer in csrc/lb200_internal.h): R ranks, L lanes per
rank, 3L exchange buffers per rank, epoch e in buffer e % 3L; batches of steps run on a rank's main stream or fork from / join into it,
and the consumer of a batch's LAST step reads its buffer on the main stream before the next batch starts.

A random scheduler interleaves everything that stream order allows (lanes of one rank progress independently, ranks drift apart) and the
model asserts what the kernels rely on: a consumer always finds, in every slab of its buffer, the rows of exactly the epoch it waits for
(no producer overwrites a buffer early), and the system never deadlocks."""
import random

import pytest


def simulate(ranks, lanes, batches, rng):
    """Each batch is dispatched the way lb200_culling_cull_exchange_n does it (a single lb200_culling_cull_exchange is a batch of one):
    - lanes >= 2 and n >= 2: fused steps, epoch e on lane e % L — the cull of e first waits for the flags of e - 2L, then stores its
      records while one of its warps publishes the lane's PREVIOUS epoch (either order); the batch ends with publish + wait of every
      lane's last epoch;
    - otherwise: two-kernel steps on the main stream — store, then publish + wait of the same epoch."""
    nbuf = 3 * lanes
    # rows[r][b][src] = epoch whose rows rank `src` last stored into buffer b of rank r; flags likewise
    rows = [[[0] * ranks for _ in range(nbuf)] for _ in range(ranks)]
    flags = [[[0] * ranks for _ in range(nbuf)] for _ in range(ranks)]
    # per rank: a list of streams; stream 0 = main.  Each op = (kind, epoch); lanes get ops between fork and join markers.
    # Build per-rank programs as dependency graphs: op ids with predecessor lists.
    progs = []
    for r in range(ranks):
        ops, last_on = [], {}   # last_on[stream] = id of the previous op on that stream

        def add(stream, kind, epoch, extra=()):
            deps = [last_on[stream]] if stream in last_on else []
            deps += list(extra)
            ops.append(dict(stream=stream, kind=kind, epoch=epoch, deps=deps, done=False))
            last_on[stream] = len(ops) - 1
            return len(ops) - 1
        epoch = 0
        for n in batches:
            if lanes < 2 or n < 2:
                for _ in range(n):
                    epoch += 1
                    for kind in ("store", "publish", "wait"):
                        add("main", kind, epoch)
                add("main", "consume", epoch)
                continue
            fork = add("main", "fork", 0)
            used = set()
            owed = {}  # lane -> its previous epoch, published by the lane's next cull or at the end of the batch
            for _ in range(n):
                epoch += 1
                lane = ("lane", epoch % lanes)
                first = lane not in used
                used.add(lane)
                if epoch - 2 * lanes >= 1:
                    add(lane, "wait", epoch - 2 * lanes, extra=[fork] if first else ())
                    first = False
                todo = [("store", epoch)] + ([("publish", owed.pop(lane))] if lane in owed else [])
                rng.shuffle(todo)
                for kind, ep in todo:
                    add(lane, kind, ep, extra=[fork] if first else ())
                    first = False
                owed[lane] = epoch
            for lane in list(owed):  # the trailing publish + wait of every lane's last epoch
                ep = owed.pop(lane)
                add(lane, "publish", ep)
                add(lane, "wait", ep)
            add("main", "join", 0, extra=[last_on[l] for l in used])
            add("main", "consume", epoch)  # the out parameters describe the LAST step of the batch
        progs.append(ops)
    pending = sum(len(p) for p in progs)
    steps = 0
    while pending:
        ready = []
        for r, ops in enumerate(progs):
            for i, op in enumerate(ops):
                if op["done"] or not all(ops[d]["done"] for d in op["deps"]):
                    continue
                if op["kind"] == "wait" and not all(flags[r][op["epoch"] % nbuf][src] >= op["epoch"] for src in range(ranks)):
                    continue  # the wait kernel keeps spinning
                ready.append((r, i))
        assert ready, "deadlock"
        r, i = rng.choice(ready)
        op = progs[r][i]
        e = op["epoch"]
        if op["kind"] == "store":
            for dst in range(ranks):
                rows[dst][e % nbuf][r] = e
        elif op["kind"] == "publish":
            for dst in range(ranks):
                flags[dst][e % nbuf][r] = max(flags[dst][e % nbuf][r], e)
        elif op["kind"] == "consume":
            assert rows[r][e % nbuf] == [e] * ranks, (r, e, rows[r][e % nbuf])
        op["done"] = True
        pending -= 1
        steps += 1
    return steps


def _batches(rng, longest):
    # single steps (two-kernel steps on the main stream) between batches of fused steps, as callers mix cull_exchange and cull_exchange_n
    return [rng.choice((1, rng.randint(2, longest))) for _ in range(rng.randint(2, 6))]


@pytest.mark.parametrize("ranks,lanes", [(2, 1), (2, 2), (2, 3), (3, 3), (8, 3), (4, 4), (8, 6), (8, 8)])
def test_no_early_overwrite_and_no_deadlock(ranks, lanes):
    rng = random.Random(1000 * ranks + lanes)
    for trial in range(12 if ranks < 8 else 3):
        simulate(ranks, lanes, _batches(rng, 20), rng)


@pytest.mark.parametrize("ranks,lanes", [(2, 1), (2, 2), (2, 3), (3, 3), (8, 3), (4, 4), (8, 8)])
def test_fused_publish_no_early_overwrite_and_no_deadlock(ranks, lanes):
    """Long batches back to back, a single step only where a batch size of 1 is drawn: with two or more lanes nearly every step is
    fused, so between a fast rank and a slow one there is little but the fused steps' flow control and the batches' closing waits."""
    rng = random.Random(53 * ranks + lanes)
    for trial in range(12 if ranks < 8 else 3):
        batches = [rng.randint(1, 20) for _ in range(rng.randint(2, 5))]
        simulate(ranks, lanes, batches, rng)


def _broken(replace, by):
    src = __import__("inspect").getsource(simulate)
    assert replace in src
    g = dict(simulate.__globals__)
    exec(src.replace(replace, by), g)
    return g["simulate"]


def test_the_model_catches_a_fused_form_without_its_flow_control():
    """Without the wait for e - 2L inside the cull a fast rank laps a slow one and overwrites the slab its consumer is about to read."""
    broken = _broken("if epoch - 2 * lanes >= 1:", "if False:")
    failures = 0
    for seed in range(80):
        try:
            broken(2, 2, [9, 9, 9], random.Random(seed))
        except AssertionError:
            failures += 1
    assert failures > 0


def test_the_model_catches_too_few_buffers():
    """Sanity of the model itself: with 2L buffers instead of 3L a fast rank does overwrite rows a slow rank has not consumed."""
    broken = _broken("nbuf = 3 * lanes", "nbuf = 2 * lanes")
    failures = 0
    for seed in range(80):
        try:
            broken(2, 2, [9, 9, 9], random.Random(seed))
        except AssertionError:
            failures += 1
    assert failures > 0
