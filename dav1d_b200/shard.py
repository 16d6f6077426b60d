"""Frame sharding over GPUs (SURVEY.md §8e): frame n is reconstructed by rank n mod G — the device-side analogue of
dav1d's frame threads (`n_fc`) — and frame n predicts from the restored pictures of frames n-1 and n-2, which other
ranks own. The dependency rule is dav1d's check_tile (reference src/thread_task.c:393-436): a band of frame n may start
once each reference has progressed past the lowest row the band reads (`lowest_pixel`, :415; progress counters
src/picture.h:52-63). Here a frame job is cut into horizontal bands (b200_frame_run_band); after each band the
producer PUTS the rows that became final into the consumers' landing buffers over NVLink peer memory and raises their
progress flag; the consumer's stream waits for exactly the flag value its band needs. No collective, no host
synchronisation on the data path; `torch.distributed` only exchanges the IPC handles (and carries the CPU tests).
Frames with intra blocks (mixed inter frames, key frames) are banded like pure inter frames: FrameBuffers(band_rows=...) gives
their bands the buffer in which each band saves its pre-filter bottom rows for the next band's intra prediction.

    PeerExchange   CUDA IPC peer pointers + copy engine puts + stream-ordered flags (the product path on GPUs)
    DistExchange   the same schedule over torch.distributed isend / recv (gloo, in the CPU tests on the host emulator)
"""
import ctypes as C

import numpy as np

K_SLOTS = 2            # landing buffers per (consumer, reference distance): frame seq of a producer lands in slot seq % K_SLOTS
FLAG_BYTES = 4096      # flag area at the head of every rank's arena
SEQ_SHIFT = 10         # progress flag value = (producer frame seq << SEQ_SHIFT) + bands done


def frame_owner(n, world):
    return n % world


def rows_to_bytes(S, plane, r0, r1):
    """byte range [a, b) inside a picture allocation that holds rows [r0, r1) of `plane` (whole rows, pitch included)"""
    px = S["pic"].itemsize
    o, st = S["off"][plane], S["stride"][plane]
    return (o + r0 * st) * px, (o + r1 * st) * px


class PeerExchange:
    """One arena per rank (flags + K_SLOTS landing pictures per reference distance), exported with CUDA IPC; every rank
    maps the arenas of the ranks it sends to (rank + d) and of those it acknowledges to (rank - d)."""

    def __init__(self, lib, dist, rank, world, pic_bytes, n_refs):
        self.lib, self.rank, self.world, self.n_refs = lib, rank, world, n_refs
        self.pic_bytes = pic_bytes = (pic_bytes + 255) & ~255      # slot pitch: landing buffers keep the source's alignment (b200_put_rows)
        self.arena_bytes = FLAG_BYTES + n_refs * K_SLOTS * pic_bytes
        self.arena = lib.b200_dev_alloc(self.arena_bytes)
        if not self.arena:
            raise RuntimeError("b200_dev_alloc: " + lib.b200_last_error().decode())
        lib.check(lib.b200_dev_memset(self.arena, 0, FLAG_BYTES, None), "b200_dev_memset")
        lib.check(lib.b200_frame_wait(None), "b200_frame_wait")
        h = (C.c_uint8 * 64)()
        lib.check(lib.b200_ipc_export(self.arena, h), "b200_ipc_export")
        handles = [None] * world
        dist.all_gather_object(handles, bytes(h))
        self.peer = {rank: self.arena}
        for d in range(1, n_refs + 1):
            for r in ((rank + d) % world, (rank - d) % world):
                if r not in self.peer:
                    hb = (C.c_uint8 * 64).from_buffer_copy(handles[r])
                    p = lib.b200_ipc_open(hb)
                    if not p:
                        raise RuntimeError("b200_ipc_open(rank %d): %s" % (r, lib.b200_last_error().decode()))
                    self.peer[r] = p
        dist.barrier()

    # layout inside an arena (the same on every rank)
    def landing_off(self, d, slot):
        return FLAG_BYTES + ((d - 1) * K_SLOTS + slot) * self.pic_bytes

    @staticmethod
    def prog_flag_off(d):          # written by the producer at distance d, waited on by the owner
        return 64 * d

    @staticmethod
    def ack_flag_off(d):           # written by the consumer at distance d ("frame seq consumed"), waited on by the owner
        return 2048 + 64 * d

    def landing_ptr(self, d, slot):
        return self.arena + self.landing_off(d, slot)

    def put(self, consumer, d, slot, a, b, src_ptr, stream):
        self.lib.check(self.lib.b200_copy_async(self.peer[consumer] + self.landing_off(d, slot) + a, src_ptr + a, b - a, stream), "b200_copy_async")

    def signal_progress(self, consumer, d, value, stream):
        self.lib.check(self.lib.b200_flag_signal(self.peer[consumer] + self.prog_flag_off(d), value, stream), "b200_flag_signal")

    def put_band(self, consumers, slot, ranges, src_ptr, seq, bands, base, counter, stream):
        """one band's put to all its consumers in one launch (b200_put_rows): `ranges` byte ranges of the picture at src_ptr
        into landing slot `slot` of every (d, rank) in `consumers`, then their progress flags = (seq << SEQ_SHIFT) + bands
        (seq read from the device word `base` when given: graph replay)"""
        from . import _lib
        assert len(consumers) <= 2 and len(ranges) <= 3
        R = (_lib.PutRange * len(ranges))()
        for i, (a, b) in enumerate(ranges):
            R[i].src = src_ptr + a
            R[i].bytes = b - a
            for j, (d, c) in enumerate(consumers):
                R[i].dst[j] = self.peer[c] + self.landing_off(d, slot) + a
        F = (_lib.PutFlag * len(consumers))()
        for j, (d, c) in enumerate(consumers):
            F[j].flag = self.peer[c] + self.prog_flag_off(d)
            if base is not None:
                F[j].base, F[j].sub, F[j].shift, F[j].add = base, 0, SEQ_SHIFT, bands
            else:
                F[j].base, F[j].add = None, (seq << SEQ_SHIFT) + bands
        self.lib.check(self.lib.b200_put_rows(R, len(ranges), F, len(consumers), counter, stream), "b200_put_rows")

    def wait_progress(self, d, value, stream, **_):
        self.lib.check(self.lib.b200_flag_wait_geq(self.arena + self.prog_flag_off(d), value, stream), "b200_flag_wait_geq")

    def signal_ack(self, producer, d, value, stream):
        self.lib.check(self.lib.b200_flag_signal(self.peer[producer] + self.ack_flag_off(d), value, stream), "b200_flag_signal")

    def wait_ack(self, d, value, stream):
        self.lib.check(self.lib.b200_flag_wait_geq(self.arena + self.ack_flag_off(d), value, stream), "b200_flag_wait_geq")

    # the same with values derived on the device from a sequence word (graph replay; see GopPipeline):
    # progress value = ((seq - wrap) << SEQ_SHIFT) + bands, acknowledgement value = seq - wrap + 1
    def signal_progress_rel(self, consumer, d, base, bands, stream):
        self.lib.check(self.lib.b200_flag_signal_rel(self.peer[consumer] + self.prog_flag_off(d), base, 0, SEQ_SHIFT, bands, stream), "b200_flag_signal_rel")

    def wait_progress_rel(self, d, base, wrap, bands, stream):
        self.lib.check(self.lib.b200_flag_wait_geq_rel(self.arena + self.prog_flag_off(d), base, wrap, SEQ_SHIFT, bands, stream), "b200_flag_wait_geq_rel")

    def signal_ack_rel(self, producer, d, base, wrap, stream):
        self.lib.check(self.lib.b200_flag_signal_rel(self.peer[producer] + self.ack_flag_off(d), base, wrap, 0, 1, stream), "b200_flag_signal_rel")

    def wait_ack_rel(self, d, base, back, add, stream):
        self.lib.check(self.lib.b200_flag_wait_geq_rel(self.arena + self.ack_flag_off(d), base, back, 0, add, stream), "b200_flag_wait_geq_rel")

    def close(self):
        for r, p in self.peer.items():
            if r != self.rank:
                self.lib.b200_ipc_close(p)
        self.lib.b200_dev_free(self.arena)
        self.peer = {}


class DistExchange:
    """The same puts / progress waits as messages: put = isend of the byte range, wait_progress = blocking recv of the
    producer's messages until the flag value is reached. Works on numpy 'device' memory (host emulator, gloo) and is
    what the gloo tests run. Only valid where a band has finished when run_band returns (the emulator): a message is
    received when its consumer asks for it, so a slot's previous occupant has been consumed by then and the
    acknowledgements are implicit."""

    def __init__(self, dist, rank, world, pic_bytes, n_refs, as_tensor, new_buffer):
        self.dist, self.rank, self.world, self.n_refs, self.pic_bytes = dist, rank, world, n_refs, pic_bytes
        self.as_tensor = as_tensor
        self.land = {(d, s): new_buffer(pic_bytes) for d in range(1, n_refs + 1) for s in range(K_SLOTS)}   # (keep, ptr)
        self.have = {d: 0 for d in range(1, n_refs + 1)}          # flag value reached per distance
        self.plan = {d: [] for d in range(1, n_refs + 1)}         # messages the producer at distance d will send, in order
        self.pending = []

    def landing_ptr(self, d, slot):
        return self.land[(d, slot)][1]

    def expect(self, d, slot, value, ranges):
        """consumer-side mirror of the producer's put sequence (both sides derive it from the same band plan)"""
        self.plan[d].append((slot, value, ranges))

    def put(self, consumer, d, slot, a, b, src_ptr, stream, src_keep=None):
        t = self.as_tensor(src_keep)[a:b]
        self.pending.append(self.dist.isend(t, dst=consumer))

    def signal_progress(self, consumer, d, value, stream):
        pass                                   # the arrival of the band's messages is the signal

    def wait_progress(self, d, value, stream, **_):
        producer = (self.rank - d) % self.world
        while self.have[d] < value:
            slot, v, ranges = self.plan[d].pop(0)
            for a, b in ranges:
                self.dist.recv(self.as_tensor(self.land[(d, slot)][0])[a:b], src=producer)
            self.have[d] = v

    def signal_ack(self, producer, d, value, stream):
        pass

    def wait_ack(self, d, value, stream):
        pass

    def close(self):
        for d in self.plan:                    # drain what the producers sent but no band asked for
            if self.plan[d]:
                self.wait_progress(d, self.plan[d][-1][1], None)
        for w in self.pending:
            w.wait()
        self.pending = []


class GopPipeline:
    """This rank's share of a dependent group of pictures. Frame `seq` of this rank is global frame n = seq * world + rank;
    it is decoded in set seq % n_sets (a FrameBuffers with band plan) and predicts from frames n-1 .. n-n_refs.

    sets: FrameBuffers (band_rows set), all of one geometry. exchange: PeerExchange / DistExchange / None (world == 1).
    graphs: from a set's second frame on, the frame's whole schedule (bands, waits, puts, host copies) is replayed as ONE
    CUDA graph launch; what changes from frame to frame — the flag values — is derived on the device from the set's
    sequence word (b200_flag_*_rel). Needs an even number of sets (a set then always uses the same landing slots)."""

    def __init__(self, lib, rank, world, sets, exchange=None, n_refs=2, n_streams=1, host_io=False, n_total=None, graphs=False):
        self.n_total = n_total          # frames in the group of pictures (None: endless stream): later frames do not exist as consumers
        self.lib, self.rank, self.world, self.sets, self.x, self.n_refs = lib, rank, world, sets, exchange, n_refs
        self.n_sets = len(sets)
        # sets are reused round-robin in an endless stream: a set must not be overwritten while later frames still predict from
        # it; a finite group of pictures that keeps every owned frame in a set of its own (decode_gop) never reuses one
        reused = n_total is None or len(range(rank, n_total, world)) > self.n_sets
        assert not reused or self.n_sets * world > n_refs, "a set would be overwritten while later frames still predict from it"
        fb = sets[0]
        self.S = fb.S
        self.nb = fb.n_bands()
        assert self.nb >= 1 and all(s.n_bands() == self.nb for s in sets)
        self.ref_name = fb.ref_name
        self.host_io = False
        A = fb.alloc
        # streams that may sit in a flag wait must not share a hardware work queue with the streams that feed the peers:
        # the package sets CUDA_DEVICE_MAX_CONNECTIONS=32 before CUDA starts (dav1d_b200/__init__.py)
        self.streams = [A.new_stream() for _ in range(max(1, n_streams))]          # (keep, handle)
        assert self.n_sets % len(self.streams) == 0, "a set must always run on the same stream"
        self.copy_stream = A.new_stream() if world > 1 else (None, None)
        # a banded frame runs as two chains: the reconstruction of band k+1 beside the post filters of band k (every band is
        # a dozen small dependent launches, each paying launch latency and drain: the chain length, not the work, sets
        # the pace of a band, so bands run one after the other on one stream cost far more than the unbanded frame)
        self.post_streams = [A.new_stream() for _ in self.streams] if self.nb > 1 else None
        # progress after each band, per plane class (luma, chroma): what a consumer's `need` is compared with
        self.prog = np.array([[fb.band_progress(k, 0), fb.band_progress(k, 1)] for k in range(self.nb)], np.int64)
        # events: per set and band (local consumers on another stream), per set "frame done", "puts done"
        ev = lib.b200_event_create
        self.ev_band = [[ev() for _ in range(self.nb)] for _ in sets] if len(self.streams) > 1 else None
        self.ev_done = [ev() for _ in sets]
        self.ev_puts = [ev() for _ in sets] if world > 1 else None
        self.ev_fork = [ev() for _ in sets]
        self.ev_recon = [ev() for _ in sets]
        self.ev_post = [ev() for _ in sets]
        self.ev_up = [ev() for _ in sets]
        self.ev_down = [ev() for _ in sets]
        self.submitted = 0
        self.set_seq = [-1] * self.n_sets
        self.bytes_put = 0
        self.put_bytes_per_frame = 0
        self.up_stream = self.down_stream = (None, None)
        self.graphs = bool(graphs)
        self.graph = [None] * self.n_sets
        self.last_replayed = [False] * self.n_sets
        self.words = None
        self.aux_words = lib.b200_dev_alloc(64 * max(self.n_sets, 1))      # per set: CTA counter of its put kernel
        lib.check(lib.b200_dev_memset(self.aux_words, 0, 64 * max(self.n_sets, 1), None), "b200_dev_memset")
        lib.check(lib.b200_frame_wait(None), "b200_frame_wait")
        if self.graphs:
            assert n_total is None, "graph replay is for endless streams (every later frame of a set looks the same)"
            assert self.n_sets % K_SLOTS == 0 or world == 1, "graph replay needs a set to always use the same landing slots"
            self.words = lib.b200_dev_alloc(8192)        # per set: sequence word at 64 * set, local progress flag at 4096 + 64 * set
            lib.check(lib.b200_dev_memset(self.words, 0, 8192, None), "b200_dev_memset")
            lib.check(lib.b200_frame_wait(None), "b200_frame_wait")
        if host_io:
            self.enable_host_io()

    def seq_word(self, si):
        return self.words + 64 * si

    def local_flag(self, si):
        return self.words + 4096 + 64 * si

    def put_counter(self, si):
        return self.aux_words + 64 * si

    def enable_host_io(self):
        """end-to-end mode: every frame's records come from pinned host memory (own upload stream, so that frame n+1's
        records travel while frame n is being reconstructed) and its output picture goes back to the host (own download stream)"""
        A = self.sets[0].alloc
        for s in self.sets:
            if not getattr(s, "_host", None):
                s.prepare_host(); s._host = True
        self.up_stream, self.down_stream = A.new_stream(), A.new_stream()
        self.host_io = True
        for g in self.graph:                      # the captured schedules did not contain the copies
            if g:
                self.lib.b200_graph_destroy(g)
        self.graph = [None] * self.n_sets

    def band_needed(self, need_luma, need_chroma):
        """first band of the producer after which rows [0, need) of both plane classes are final"""
        if need_luma <= 0 and need_chroma <= 0:
            return -1
        ok = (self.prog[:, 0] >= need_luma) & (self.prog[:, 1] >= need_chroma)
        return int(np.argmax(ok))                        # the last band always satisfies it

    def ref_source(self, n, d):
        """where frame n's reference at distance d lives on this rank: (kind, ...)"""
        m = n - d
        if m < 0:
            return ("own", None)
        owner, mseq = m % self.world, m // self.world
        if owner == self.rank:
            return ("local", mseq)
        return ("remote", mseq)

    def submit(self):
        """enqueue this rank's next frame (all its bands, waits and puts); returns its local sequence number"""
        lib, world, rank = self.lib, self.world, self.rank
        seq = self.submitted
        self.submitted += 1
        si = seq % self.n_sets
        sidx = seq % len(self.streams)
        st = self.streams[sidx][1]
        # ---- the set is free again: its previous frame finished, its puts left, nobody predicts from it any more
        # (always outside a captured graph: these are dependencies on other frames' work)
        if self.set_seq[si] >= 0:
            prev = self.set_seq[si]
            replayed = self.last_replayed[si]              # its last frame ran as a graph: puts and host copies were joined inside it
            if world > 1 and not replayed:
                lib.check(lib.b200_stream_wait_event(st, self.ev_puts[si]), "wait")
            for d in range(1, self.n_refs + 1):                 # local frames that predicted from it
                r = (prev * world + rank) + d
                if r % world == rank:
                    rs = r // world
                    if rs < seq and (rs % len(self.streams)) != sidx:
                        lib.check(lib.b200_stream_wait_event(st, self.ev_done[rs % self.n_sets]), "wait")
            if self.host_io and not replayed:
                lib.check(lib.b200_stream_wait_event(st, self.ev_down[si]), "wait")     # its output picture has left
        replay = self.graphs and self.set_seq[si] >= 0
        self.last_replayed[si] = replay
        self.set_seq[si] = seq
        if replay:
            if self.graph[si] is None:
                before = self.bytes_put
                lib.check(lib.b200_graph_begin(st), "b200_graph_begin")
                self._enqueue(seq, st, sidx, rel=True)
                g = lib.b200_graph_end(st)
                if not g:
                    raise RuntimeError("b200_graph_end: " + lib.b200_last_error().decode())
                self.graph[si] = g
                self.put_bytes_per_frame = self.bytes_put - before
            else:
                self.bytes_put += self.put_bytes_per_frame
            lib.check(lib.b200_flag_signal(self.seq_word(si), seq, st), "b200_flag_signal")
            lib.check(lib.b200_graph_launch(self.graph[si], st), "b200_graph_launch")
        else:
            self._enqueue(seq, st, sidx, rel=False)
        lib.check(lib.b200_event_record(self.ev_done[si], st), "record")
        return seq

    def _enqueue(self, seq, st, sidx, rel):
        """one frame's schedule on stream st. rel: flag values come from the set's sequence word on the device (capturable)"""
        lib, x, world, rank = self.lib, self.x, self.world, self.rank
        n = seq * world + rank
        si = seq % self.n_sets
        fb = self.sets[si]
        multi = len(self.streams) > 1
        base = self.seq_word(si) if rel else None
        # ---- reference pointers
        srcs = []
        for d in range(1, self.n_refs + 1):
            kind, mseq = self.ref_source(n, d)
            srcs.append((kind, mseq))
            if kind == "local":
                fb.job.mc.ref[d - 1] = self.sets[mseq % self.n_sets].picture_ptr(self.ref_name)
            elif kind == "remote":
                fb.job.mc.ref[d - 1] = x.landing_ptr(d, mseq % K_SLOTS)
            else:
                assert not rel
                fb.job.mc.ref[d - 1] = fb.keep["ref%d" % (d - 1)][1]
        fork = lambda other: (lib.check(lib.b200_event_record(self.ev_fork[si], st), "record"),
                              lib.check(lib.b200_stream_wait_event(other, self.ev_fork[si]), "wait"))
        if self.host_io:
            us = self.up_stream[1]
            if rel:
                fork(us)                                        # inside a graph the copies hang off the frame's own stream
            else:
                lib.check(lib.b200_stream_wait_event(us, self.ev_done[si]), "wait")     # the set's previous frame no longer reads its records
            for u in fb._ups:
                lib.check(lib.b200_copy_async(u.dev, u.host, u.bytes, us), "h2d")
            lib.check(lib.b200_event_record(self.ev_up[si], us), "record")
            lib.check(lib.b200_stream_wait_event(st, self.ev_up[si]), "wait")
        consumers = [(d, (rank + d) % world) for d in range(1, self.n_refs + 1)
                     if (rank + d) % world != rank and (self.n_total is None or n + d < self.n_total)] if world > 1 else []
        if isinstance(x, DistExchange):       # tell the exchange what the producers of my references will send
            for d in range(1, self.n_refs + 1):
                if srcs[d - 1][0] == "remote":
                    mseq = srcs[d - 1][1]
                    for k in range(self.nb):
                        x.expect(d, mseq % K_SLOTS, (mseq << SEQ_SHIFT) + k + 1, self._band_ranges(k))
        waited = [-1] * (self.n_refs + 1)
        cs = self.copy_stream[1]
        forked_copy = False
        ps = self.post_streams[sidx][1] if self.post_streams is not None else None      # post-filter chain (None: one chain)
        if ps is not None and ps == st:
            ps = None
        fork_from = lambda src, other: (lib.check(lib.b200_event_record(self.ev_fork[si], src), "record"),
                                        lib.check(lib.b200_stream_wait_event(other, self.ev_fork[si]), "wait"))
        for k in range(self.nb):
            # ---- dependencies of band k: each reference must be final down to the lowest row the band reads
            for d in range(1, self.n_refs + 1):
                kind, mseq = srcs[d - 1]
                if kind == "own":
                    continue
                kn = self.band_needed(int(fb.band_need[k, d - 1, 0]), int(fb.band_need[k, d - 1, 1]))
                if kn <= waited[d]:
                    continue
                waited[d] = kn
                wrap = seq - mseq
                if kind == "local":
                    if (mseq % len(self.streams)) != sidx:
                        if rel:
                            lib.check(lib.b200_flag_wait_geq_rel(self.local_flag(mseq % self.n_sets), base, wrap, SEQ_SHIFT, kn + 1, st), "wait")
                        else:
                            lib.check(lib.b200_stream_wait_event(st, self.ev_band[mseq % self.n_sets][kn]), "wait")
                elif rel:
                    x.wait_progress_rel(d, base, wrap, kn + 1, st)
                else:
                    x.wait_progress(d, (mseq << SEQ_SHIFT) + kn + 1, st)
            if ps is None:
                fb.run_band(k, st)
                qs = st                     # the stream on which band k's restored rows are final
            else:
                fb.run_band_phase(k, 1, st)
                lib.check(lib.b200_event_record(self.ev_recon[si], st), "record")
                lib.check(lib.b200_stream_wait_event(ps, self.ev_recon[si]), "wait")
                fb.run_band_phase(k, 2, ps)
                qs = ps
            if multi:
                if self.graphs:     # local consumers on the other stream wait on a flag (events recorded inside a graph are not visible outside)
                    if rel:
                        lib.check(lib.b200_flag_signal_rel(self.local_flag(si), base, 0, SEQ_SHIFT, k + 1, qs), "signal")
                    else:
                        lib.check(lib.b200_flag_signal(self.local_flag(si), (seq << SEQ_SHIFT) + k + 1, qs), "signal")
                if not rel:
                    lib.check(lib.b200_event_record(self.ev_band[si][k], qs), "record")
            # ---- put the rows that became final into the consumers' landing buffers, then raise their flag
            if consumers:
                fork_from(qs, cs)
                forked_copy = True
                src_keep, src_ptr = fb.keep[self.ref_name]
                if k == 0:                          # the slots' previous occupants have been consumed
                    for d, c in consumers:
                        if rel:
                            x.wait_ack_rel(d, base, K_SLOTS, 1, cs)
                        elif seq >= K_SLOTS:
                            x.wait_ack(d, seq - K_SLOTS + 1, cs)
                ranges = self._band_ranges(k)
                self.bytes_put += sum(b - a for a, b in ranges) * len(consumers)
                if isinstance(x, DistExchange):
                    for d, c in consumers:
                        for a, b in ranges:
                            x.put(c, d, seq % K_SLOTS, a, b, src_ptr, cs, src_keep=src_keep)
                        x.signal_progress(c, d, (seq << SEQ_SHIFT) + k + 1, cs)
                else:       # one launch: rows to every consumer over NVLink, then their flags
                    x.put_band(consumers, seq % K_SLOTS, ranges, src_ptr, seq, k + 1, base, self.put_counter(si), cs)
        # ---- the frame is enqueued: acknowledge the references (their slots may be overwritten once this point is reached)
        for d in range(1, self.n_refs + 1):
            kind, mseq = srcs[d - 1]
            if kind == "remote":
                if rel:
                    x.signal_ack_rel((rank - d) % world, d, base, seq - mseq, st)
                else:
                    x.signal_ack((rank - d) % world, d, mseq + 1, st)
        if ps is not None:                  # the post chain joins: what follows on st (acknowledged above: only the
            lib.check(lib.b200_event_record(self.ev_post[si], ps), "record")      # reconstruction reads the references)
            lib.check(lib.b200_stream_wait_event(st, self.ev_post[si]), "wait")
        if self.host_io:
            ds = self.down_stream[1]
            fork(ds)
            for dn in fb._downs:
                lib.check(lib.b200_copy_async(dn.host, dn.dev, dn.bytes, ds), "d2h")
            lib.check(lib.b200_event_record(self.ev_down[si], ds), "record")
            if rel:
                lib.check(lib.b200_stream_wait_event(st, self.ev_down[si]), "wait")       # join: a graph has one end
        if world > 1:
            if forked_copy or not rel:
                lib.check(lib.b200_event_record(self.ev_puts[si], cs), "record")
            if rel and forked_copy:
                lib.check(lib.b200_stream_wait_event(st, self.ev_puts[si]), "wait")       # join

    def _band_ranges(self, k):
        """byte ranges of the restored picture that became final with band k (per plane: rows [progress(k-1), progress(k)))"""
        out = []
        for pl in range(3):
            cls = 1 if pl else 0
            r0 = int(self.prog[k - 1, cls]) if k else 0
            r1 = int(self.prog[k, cls])
            if r1 > r0:
                out.append(rows_to_bytes(self.S, pl, r0, r1))
        return out

    def sync(self):
        for _, h in self.streams:
            self.lib.check(self.lib.b200_frame_wait(h), "b200_frame_wait")
        for h in [self.copy_stream[1], self.up_stream[1], self.down_stream[1]] + [p[1] for p in (self.post_streams or [])]:
            if h is not None:
                self.lib.check(self.lib.b200_frame_wait(h), "b200_frame_wait")

    def output(self, seq, name=None):
        return self.sets[seq % self.n_sets].output(name or self.ref_name)


def decode_gop(frames, make_buffers, dist, rank, world, lib, exchange="peer", band_rows=64, n_refs=2, n_sets=None, n_streams=1,
               as_tensor=None, new_buffer=None):
    """Reconstruct `frames` (synthetic frame dicts, decode order): frame k on rank k mod world, predicting from the restored
    pictures of frames k-1 and k-2 (its own synthetic references stand in for pictures before the GOP). Every rank returns
    {k: restored picture} for the frames it owns. make_buffers(S, band_rows) -> FrameBuffers on this rank's device."""
    mine = [k for k in range(len(frames)) if k % world == rank]
    n_sets = n_sets or max(len(mine), 1)
    assert n_sets >= len(mine), "decode_gop keeps every owned frame resident"
    sets = [make_buffers(frames[k], band_rows) for k in mine] or [make_buffers(frames[0], band_rows)]
    x = None
    pic_bytes = frames[0]["pic"].nbytes
    if world > 1:
        if exchange == "peer":
            x = PeerExchange(lib, dist, rank, world, pic_bytes, n_refs)
        else:
            x = DistExchange(dist, rank, world, pic_bytes, n_refs, as_tensor, new_buffer)
    pipe = GopPipeline(lib, rank, world, sets, exchange=x, n_refs=n_refs, n_streams=n_streams, n_total=len(frames))
    for _ in mine:
        pipe.submit()
    pipe.sync()
    if x is not None:
        if dist is not None:
            dist.barrier()
        x.close()
    return {k: pipe.output(i).copy() for i, k in enumerate(mine)}
