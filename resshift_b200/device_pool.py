"""Device pool: one process drives several GPUs (``ResShiftSampler(devices=...)`` or ``RS_DEVICES``), bit-identical to
one GPU (DESIGN.md §6).

Every entry of the pool is a replica: a copy of the denoiser and the VQ-GAN on one device, with its own engine, arena,
plans and CUDA stream, driven by its own host thread.  The sampler's main thread walks the work units of a chunk in
one-GPU order and draws each unit's noise on the primary device (the first entry), exactly as a one-GPU run does; the
units then run on whichever replica is free.  A unit's output does not depend on the device that runs it, so the tiles
that come back to the primary are the one-GPU tiles.  With fewer units than replicas, the chunk's schedule
(``parallel.unit_schedule``) runs each unit on a team of replicas that splits its VQ-GAN bottleneck attention; the rows
are exchanged in process by ``TeamExchange``.

The library's kernels pick their tile configurations from the device's SM count, so a pool refuses devices that differ
in SM count or compute capability.
"""
from __future__ import annotations

import os
import queue
import threading
from contextlib import nullcontext
from typing import Callable, List, Optional, Sequence

import torch

from .parallel import attention_row_ranges


def parse_devices(spec, count: int) -> List[int]:
    """Device indices of a pool: ``"all"`` (every visible GPU), ``"0,2,3"``, an int, or a sequence of ints or
    ``torch.device``.  The same index may appear more than once (one replica per entry).  Raises ValueError on an
    index that is not visible."""
    if isinstance(spec, str):
        s = spec.strip().lower()
        if s == "all":
            if count < 1:
                raise ValueError("RS_DEVICES=all: no CUDA device is visible")
            return list(range(count))
        try:
            ids = [int(tok) for tok in s.split(",")]
        except ValueError:
            raise ValueError(f"device pool {spec!r}: expected 'all' or comma-separated device indices such as '0,2,3'") from None
    elif isinstance(spec, int):
        ids = [spec]
    else:
        ids = []
        for d in spec:
            if isinstance(d, torch.device):
                if d.type != "cuda" or d.index is None:
                    raise ValueError(f"device pool entry {d}: give a CUDA device with an index")
                d = d.index
            ids.append(int(d))
    if not ids:
        raise ValueError("a device pool needs at least one device")
    for i in ids:
        if not 0 <= i < count:
            raise ValueError(f"device pool entry {i}: only {count} CUDA device(s) are visible")
    return ids


def check_identical_devices(ids: Sequence[int], properties: Callable = None) -> None:
    """Refuses a pool whose devices differ in SM count or compute capability: the conv launcher sizes its tiles and
    grids from the SM count, so such devices would not compute bit-identical results."""
    properties = properties or torch.cuda.get_device_properties
    seen = {}
    for i in ids:
        if i not in seen:
            p = properties(i)
            seen[i] = (p.multi_processor_count, p.major, p.minor, p.name)
    first = seen[ids[0]]
    for i in ids:
        if seen[i][:3] != first[:3]:
            raise ValueError(
                f"a device pool needs identical devices: cuda:{ids[0]} is {first[3]} ({first[0]} SMs, compute "
                f"capability {first[1]}.{first[2]}) but cuda:{i} is {seen[i][3]} ({seen[i][0]} SMs, compute capability "
                f"{seen[i][1]}.{seen[i][2]}); tile configurations depend on the SM count, so results would differ")


def pool_devices(devices=None, environ=None, device_count: Optional[int] = None, properties: Callable = None):
    """The device indices of ``ResShiftSampler(devices=...)``, or None for no pool.  ``devices=None`` reads
    ``RS_DEVICES``; unset or empty (and an empty ``devices``) means no pool.  Refused: a pool inside a multi-process
    run (``WORLD_SIZE > 1``), invisible devices and devices that are not identical."""
    environ = os.environ if environ is None else environ
    spec = environ.get("RS_DEVICES", "") if devices is None else devices
    if spec is None or (isinstance(spec, str) and not spec.strip()) or (isinstance(spec, (list, tuple)) and not spec):
        return None
    if int(environ.get("WORLD_SIZE", "1")) > 1:
        raise ValueError("a device pool (devices= / RS_DEVICES) drives several GPUs from one process and does not combine "
                         "with one process per GPU (WORLD_SIZE > 1): use one or the other")
    ids = parse_devices(spec, torch.cuda.device_count() if device_count is None else device_count)
    check_identical_devices(ids, properties)
    return ids


class Replica:
    """One pool entry: the models that run its units and the stream they run on.  A replica on another device than the
    primary also gets a ``link`` stream on the primary, on which its worker's copies to and from the primary run (its
    thread's current stream there), so that they never wait behind the calling thread's work on the primary."""

    def __init__(self, index: int, device: int, model, autoencoder, primary: int):
        self.index, self.device = index, torch.device("cuda", device)
        self.model, self.autoencoder = model, autoencoder
        with torch.cuda.device(self.device):
            self.stream = torch.cuda.Stream()
        self.link = None
        if device != primary:
            with torch.cuda.device(primary):
                self.link = torch.cuda.Stream()


class TeamExchange:
    """``exchange(view, row_begin, row_end)`` callables (``member(m)``) for the replicas of one attention team
    (VQModelTorch.attention_team).  Each member's thread calls its exchange after enqueuing the first half of the pass
    on its stream.  The copies are ordered by CUDA events on the members' streams:
      1. every member records ``begun`` on its stream (its rows are being computed into its view);
      2. the team meets at a barrier;
      3. for every other member o, a ``pull`` stream of this member on o's device waits for ``begun[o]`` and copies
         o's rows into a dense buffer (the row slice of an [N, T, C] view is strided when N > 1) and from there to this
         member's device; this member's stream waits for the pull stream and writes the rows into its own view;
      4. every member records ``copied``;
      5. the team meets at a second barrier;
      6. every member's stream waits for all ``copied`` events, so that no member's second half (or its next unit)
         overwrites a view that another member is still reading.
    Every read of another member's view is thus on a stream ordered after that member's ``begun``, and every write to
    this member's view is on its own stream: nothing depends on how PyTorch orders a cross-device copy internally.  The
    same path runs when members share a device.  The second barrier also keeps a member from publishing the next
    exchange's events before the others have read this one's."""

    def __init__(self, size: int):
        self.size = size
        self.barrier = threading.Barrier(size)
        self.views: List[Optional[torch.Tensor]] = [None] * size
        self.begun: List[Optional[torch.cuda.Event]] = [None] * size
        self.copied: List[Optional[torch.cuda.Event]] = [None] * size
        self.pulls: List[dict] = [{} for _ in range(size)]      # member -> {source device: stream}, one thread each

    def member(self, m: int):
        return lambda view, row_begin, row_end: self._exchange(m, view, row_begin, row_end)

    def _pull_stream(self, m: int, device: torch.device) -> torch.cuda.Stream:
        if device not in self.pulls[m]:
            with torch.cuda.device(device):
                self.pulls[m][device] = torch.cuda.Stream()
        return self.pulls[m][device]

    def _exchange(self, m: int, view: torch.Tensor, row_begin: int, row_end: int) -> None:
        ranges = attention_row_ranges(view.shape[1], self.size)
        assert ranges[m] == (row_begin, row_end), (ranges, m, row_begin, row_end)
        stream = torch.cuda.current_stream(view.device)
        self.views[m] = view
        self.begun[m] = torch.cuda.Event()
        self.begun[m].record(stream)
        self.barrier.wait()
        for o, (b, e) in enumerate(ranges):
            if o == m or e <= b:
                continue
            src = self.views[o][:, b:e]
            pull = self._pull_stream(m, src.device)
            pull.wait_event(self.begun[o])
            with torch.cuda.stream(pull):                       # (makes src's device current, pull its stream)
                dense = src.contiguous()                        # on pull, after begun[o]
                landed = dense.to(view.device, non_blocking=True)   # dense: one memcpy on pull, no temporaries
            stream.wait_stream(pull)
            landed.record_stream(stream)
            with torch.cuda.device(view.device):
                view[:, b:e].copy_(landed)                      # on this member's stream
        self.copied[m] = torch.cuda.Event()
        self.copied[m].record(stream)
        self.barrier.wait()
        for o in range(self.size):
            if o != m:
                stream.wait_event(self.copied[o])


class _Job:
    __slots__ = ("unit", "pch", "mch", "noises", "spec", "ready", "team", "keep")

    def __init__(self, unit, pch, mch, noises, spec, ready, team=None, keep=True):
        self.unit, self.pch, self.mch, self.noises, self.spec, self.ready = unit, pch, mch, noises, spec, ready
        self.team, self.keep = team, keep


class DevicePool:
    """The replicas of a ResShiftSampler and the threads that run a chunk's units on them."""

    def __init__(self, replicas: Sequence[Replica]):
        self.replicas = list(replicas)
        self.primary = self.replicas[0].device

    def run(self, sampler, lqs, masks, noise_repeat, units):
        """Runs every unit of ``units`` (ResShiftSampler._plan_units of the chunk ``lqs`` / ``masks`` on the primary
        device) and returns, per unit, its output [n * b, 3, th*sf, tw*sf] on the primary device.  Noise is drawn here,
        on the calling thread, in unit order (ResShiftSampler._unit_noises); a unit goes to the next free replica, or,
        when the chunk's schedule (ResShiftSampler._schedule) has teams, to every member of its team.  An exception in
        any worker stops the others and is raised here."""
        n = len(self.replicas)
        schedule = sampler._schedule(len(units), n)
        teams = any(e - a > 1 for a, e in schedule)
        stop = threading.Event()
        errors: List[BaseException] = []
        exchanges = [TeamExchange(e - a) for a, e in schedule] if teams else []
        lock = threading.Lock()

        def fail(exc):
            with lock:
                errors.append(exc)
            stop.set()
            for x in exchanges:
                x.barrier.abort()

        if not teams:                                           # deal units to whichever replica is free
            shared = queue.Queue(maxsize=2 * n)
            inboxes = [shared] * n
        else:                                                   # unit u runs on its team's replicas
            inboxes = [queue.Queue() for _ in range(n)]
        results: List[Optional[tuple]] = [None] * len(units)      # (output on the primary, event completing it)
        threads = [threading.Thread(target=self._work, args=(r, sampler, inboxes[r], results, stop, fail),
                                    name=f"rs-device-pool-{r}", daemon=True) for r in range(n)]
        for t in threads:
            t.start()
        main_stream = torch.cuda.current_stream(self.primary)
        try:
            for i, noises, spec in sampler._unit_noises(lqs, noise_repeat, units):
                if stop.is_set():
                    break
                pch, mch = sampler._unit_input(lqs, masks, units[i])
                ready = torch.cuda.Event()
                ready.record(main_stream)
                if not teams:
                    _put(shared, _Job(i, pch, mch, noises, spec, ready), stop)
                    continue
                a, e = schedule[i]
                for r in range(a, e):
                    team = (r - a, e - a, exchanges[i].member(r - a)) if e - a > 1 else None
                    inboxes[r].put(_Job(i, pch, mch, noises, spec, ready, team, keep=r == a))
            for r in range(n):
                if not _put(inboxes[r], None, stop):
                    break
        except BaseException as exc:                            # noqa: BLE001 — stop the workers, then re-raise below
            fail(exc)
        finally:
            for t in threads:
                t.join()
        if errors:
            raise errors[0]
        out = []
        for res, done in results:                               # read on the caller's stream from here on
            main_stream.wait_event(done)
            res.record_stream(main_stream)
            out.append(res)
        return out

    def _work(self, r, sampler, inbox, results, stop, fail):
        """Worker thread of replica ``r``.  It enqueues a unit, then waits for the one before it to finish, so the
        device always has the next unit queued while units are still dealt by actual progress (a worker holds at most
        one unit beyond the one its device is running)."""
        rep = self.replicas[r]
        try:
            torch.cuda.set_device(rep.device)
            # (entering a stream context also makes its device current: the replica's stream comes last)
            with torch.cuda.stream(rep.link) if rep.link is not None else nullcontext(), torch.cuda.stream(rep.stream):
                assert torch.cuda.current_device() == rep.device.index
                prev = None
                while True:
                    job = _get(inbox, stop)
                    if job is None:
                        return
                    res, done = self._run_job(rep, sampler, job)
                    if job.keep:
                        results[job.unit] = (res, done)
                    if prev is not None:
                        prev.synchronize()
                    prev = done
        except BaseException as exc:                            # noqa: BLE001 — handed to the calling thread
            fail(exc)
            try:                                                # let the failed unit's launches finish
                for s in (rep.stream, rep.link):
                    if s is not None:
                        s.synchronize()
            except Exception:                                   # noqa: BLE001 — the first error is what matters
                pass

    def _run_job(self, rep: Replica, sampler, job: _Job):
        """Enqueues one unit on ``rep``'s stream (the current stream of this thread): the inputs after ``job.ready``
        on the caller's stream, the output copied to the primary.  Returns the output (None for a team member other
        than the first) and an event that completes with the unit, on this thread's current stream of the primary
        (``rep.stream`` when the replica is on the primary; else ``rep.link``, which the cross-device copies ran on)."""
        primary_stream = torch.cuda.current_stream(self.primary)
        rep.stream.wait_event(job.ready)
        dev = rep.device
        pch = job.pch.to(dev, non_blocking=True)
        mch = None if job.mch is None else job.mch.to(dev, non_blocking=True)
        # (the posterior noise, if any, stays on the CPU: the first stage copies it, as the reference's encode does)
        noises = job.noises._replace(loop=job.noises.loop.to(dev, non_blocking=True))
        for t in (job.pch, job.mch, job.noises.loop):           # read on primary_stream: not reused before that
            if t is not None:
                t.record_stream(primary_stream)
        res = sampler._run_unit(pch, mch, noises, job.spec, team=job.team, replica=rep)
        res = res.to(self.primary, non_blocking=True) if job.keep else None
        done = torch.cuda.Event()
        if dev != self.primary:                                 # the unit itself ran on rep.stream
            primary_stream.wait_stream(rep.stream)
        done.record(primary_stream)
        return res, done


def _put(q: queue.Queue, item, stop: threading.Event) -> bool:
    while not stop.is_set():
        try:
            q.put(item, timeout=0.05)
            return True
        except queue.Full:
            pass
    return False


def _get(q: queue.Queue, stop: threading.Event):
    while not stop.is_set():
        try:
            return q.get(timeout=0.05)
        except queue.Empty:
            pass
    return None
