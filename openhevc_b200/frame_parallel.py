"""Frame-parallel decoding of a random-access (hierarchical-B, GOP 8) stream over N GPUs.

Mirror of the reference's frame threads (libavcodec/pthread_frame.c; context i <-> GPU i mod N) at the
only granularity at which this path shards (SURVEY.md §8e): whole pictures.  Inside a GOP the seven B pictures only reference pictures of the same GOP and the two
surrounding anchors.  Ownership is by INTRA PERIOD (4 GOPs, 32 pictures: period q -> rank q mod N): the anchor
chain I -> P -> P -> P of a period stays on one GPU, and the ONE exchange step is the last anchor of a period,
which the seven leading B pictures of the next period reference (open GOP): the analogue of
ff_thread_report_progress(&ref->tf, INT_MAX), hevc.c:4026, as one NCCL send / receive over NVLink to the single
GPU that reads it (24.9 MB per 32 pictures at 4K Main10), on a side stream, off every critical path.  Nothing
else ever leaves its GPU.

The schedule is written against a tiny backend interface so that the very same code runs
  * on GPUs  (GpuBackend: libb200hevc + torch.distributed/NCCL, CUDA events between streams), and
  * in the CPU test-suite (tests/test_frame_parallel_cpu.py: gloo, world_size 2, pictures "decoded" by the
    test oracle) -- the host logic, slot rotation and collective order are identical.
"""
from dataclasses import dataclass
from typing import List

N_ANCHOR_SLOTS = 16            # anchors rotate through slots 0..15: a slot is reused 16 GOPs later
N_B_SLOTS = 21                 # three sets of seven: consecutive GOPs do not wait for each other's B pictures (WAR on the slots);
                               # the third set is for the B pictures a period issues last (period_pictures)
N_SLOTS = N_ANCHOR_SLOTS + N_B_SLOTS
INTRA_PERIOD_GOPS = 4          # every 4th anchor is an I picture (intra period 32 pictures)

# blob indices of the 9 distinct pictures of the periodic stream
BLOB_ANCHOR_P, BLOB_ANCHOR_I, BLOB_B4, BLOB_B2, BLOB_B6, BLOB_B1, BLOB_B3, BLOB_B5, BLOB_B7 = range(9)
N_BLOBS = 9


@dataclass
class Picture:
    blob: int
    cur_slot: int
    ref_slots: List[int]
    anchor: bool


def anchor_slot(g):
    return g % N_ANCHOR_SLOTS


def gop_pictures(g, lg=None, b_set=None):
    """decode-order pictures of GOP g (POC order 8g+{8,4,2,6,1,3,5,7}) with their DPB placement.  lg: the GOP's index among the
    GOPs THIS GPU decodes (default g): DPB slots rotate per GPU, so that consecutive periods of one GPU never share a slot"""
    lg = g if lg is None else lg
    a_prev, a_cur = anchor_slot(lg - 1), anchor_slot(lg)
    b = [N_ANCHOR_SLOTS + 7 * ((lg & 1) if b_set is None else b_set) + k for k in range(7)]     # b4, b2, b6, b1, b3, b5, b7
    intra = g % INTRA_PERIOD_GOPS == 0
    return [
        Picture(BLOB_ANCHOR_I if intra else BLOB_ANCHOR_P, a_cur, [] if intra else [a_prev], True),
        Picture(BLOB_B4, b[0], [a_prev, a_cur], False),
        Picture(BLOB_B2, b[1], [a_prev, b[0]], False),
        Picture(BLOB_B6, b[2], [b[0], a_cur], False),
        Picture(BLOB_B1, b[3], [a_prev, b[1]], False),
        Picture(BLOB_B3, b[4], [b[1], b[0]], False),
        Picture(BLOB_B5, b[5], [b[0], b[2]], False),
        Picture(BLOB_B7, b[6], [b[2], a_cur], False),
    ]


def blob_specs():
    """(name, n_refs) of the distinct work lists the stream is made of"""
    return [("anchor_P", 1), ("anchor_I", 0)] + [(n, 2) for n in ("b4", "b2", "b6", "b1", "b3", "b5", "b7")]


def period_owner(q, world):
    """intra period q (INTRA_PERIOD_GOPS GOPs, 32 pictures) is decoded by rank q mod N"""
    return q % world


def period_pictures(q, k=None, n_gops=INTRA_PERIOD_GOPS):
    """The pictures of intra period q in the order its owner issues them, and which of them waits for the one picture that
    comes from another GPU.  n_gops < INTRA_PERIOD_GOPS: only the first n_gops GOPs of the period (the end of a run).

    A period starts with an I anchor, so its anchor chain I -> P -> P -> P never leaves the GPU (giving GOP g to rank g mod N
    would make every anchor wait for the previous GOP's anchor on another GPU: decode -> send -> decode in series).  The stream
    is open-GOP: the seven B pictures in front of the I anchor (output order) still reference the LAST anchor of the previous period.  They are leaves -- nothing references them -- so the owner issues them
    last, when that anchor has long arrived (it is the 4th of the 4 anchors of the neighbour's period, which runs at the same
    time).  k: index of the period among the periods of its GPU (slot rotation; default q).
    Returns [(global GOP index, Picture, needs_prev_period_anchor)]."""
    k = q if k is None else k
    g0 = q * INTRA_PERIOD_GOPS
    out, deferred = [], []
    for g in range(g0, g0 + n_gops):
        pics = gop_pictures(g, k * INTRA_PERIOD_GOPS + (g - g0), 2 if g == g0 else (g - g0) & 1)
        out.append((g, pics[0], False))
        if g == g0:
            deferred = [(g, p, True) for p in pics[1:]]
        else:
            out += [(g, p, False) for p in pics[1:]]
    return out + deferred


def run_schedule(backend, rank, world, n_gops_per_rank):
    """Issue the whole schedule (asynchronously on a GPU backend).  Returns pictures decoded by this rank.
    n_gops_per_rank GOPs per rank = n_gops_per_rank / 4 intra periods per rank; period q goes to rank q mod N.  A remainder
    cuts the last period short on one rank; with several ranks it is rounded up to a whole period, so that the GOPs decoded
    are always the first ones of the stream.  The one exchange per period: its owner receives the previous
    period's last anchor from rank - 1 and sends its own last anchor to rank + 1 (point to point: exactly one GPU ever reads it)."""
    rounds = -(-n_gops_per_rank // INTRA_PERIOD_GOPS)
    n_periods = rounds * world
    decoded = 0
    for k in range(rounds):
        q = k * world + rank
        n_gops = min(INTRA_PERIOD_GOPS, n_gops_per_rank - k * INTRA_PERIOD_GOPS) if world == 1 else INTRA_PERIOD_GOPS
        recv_slot = anchor_slot(k * INTRA_PERIOD_GOPS - 1) if (world > 1 and q > 0) else None
        send_slot = anchor_slot(k * INTRA_PERIOD_GOPS + n_gops - 1) if (world > 1 and q + 1 < n_periods) else None
        exchanged = False
        for (g, pic, needs_prev) in period_pictures(q, k, n_gops):
            if needs_prev and not exchanged:
                # the last anchor of this period is decoded (the deferred pictures come after everything else): one grouped
                # exchange, ordered on the device by the slots' hazards
                backend.exchange_anchors(send_slot, (rank + 1) % world, recv_slot, (rank - 1) % world)
                exchanged = True
            backend.decode(pic, g)
            decoded += 1
        if not exchanged:
            backend.exchange_anchors(send_slot, (rank + 1) % world, recv_slot, (rank - 1) % world)
    return decoded


class GpuBackend:
    """libb200hevc engine + NCCL.  The DPB lives in a torch tensor so that torch.distributed can address slots.
    Ordering on the device is the engine's slot-hazard tracking (include/b200hevc.h: b200_slot_begin/end_access):
    the broadcast is a reader of the anchor's slot on its owner and a writer of the slot everywhere else, on the
    communication stream, so it overlaps the B pictures of the previous GOP on the compute lanes."""

    def __init__(self, engine, dpb_tensor, slot_bytes, world, arenas_of_blob):
        import torch
        self.torch = torch
        self.eng, self.dpb, self.slot_bytes, self.world = engine, dpb_tensor, slot_bytes, world
        self.arena = arenas_of_blob
        self.compute = torch.cuda.ExternalStream(engine.lib.b200_stream(engine.h))
        self.comm = torch.cuda.Stream() if world > 1 else None
        self.bcast_bytes = 0
        if world > 1:
            # Open the point-to-point connections of the ring once, SYMMETRICALLY (every rank sends right and receives from the
            # left in one group): NCCL sets a pair's channels up at their first use and expects both ends in matching groups --
            # the schedule's first exchange is not (rank 0 only sends), which NCCL 2.28 answers with "Message truncated".
            import torch.distributed as dist
            rank = dist.get_rank()
            a, b = torch.zeros(16, device=dpb_tensor.device), torch.zeros(16, device=dpb_tensor.device)
            with torch.cuda.stream(self.comm):
                for w in dist.batch_isend_irecv([dist.P2POp(dist.isend, a, (rank + 1) % world), dist.P2POp(dist.irecv, b, (rank - 1) % world)]):
                    w.wait()
            self.comm.synchronize()

    def decode(self, pic, g=None):
        self.eng.execute(self.arena[pic.blob], pic.cur_slot, pic.ref_slots)

    def exchange_anchors(self, send_slot, dst, recv_slot, src):
        """one NCCL group: send this period's last anchor to the owner of the next period, receive the previous period's last
        anchor.  On the communication stream, inside the engine's slot-hazard protocol: a reader of the slot it sends, a writer
        of the slot it receives -- so the B pictures that need the received anchor wait for it on the device, nothing else does."""
        if send_slot is None and recv_slot is None:
            return
        torch = self.torch
        import torch.distributed as dist
        ops = []
        with torch.cuda.stream(self.comm):
            if recv_slot is not None:
                self.eng.slot_begin_access(recv_slot, self.comm.cuda_stream, True)
                ops.append(dist.P2POp(dist.irecv, self.dpb[recv_slot * self.slot_bytes:(recv_slot + 1) * self.slot_bytes], src))
            if send_slot is not None:
                self.eng.slot_begin_access(send_slot, self.comm.cuda_stream, False)
                ops.append(dist.P2POp(dist.isend, self.dpb[send_slot * self.slot_bytes:(send_slot + 1) * self.slot_bytes], dst))
            for w in dist.batch_isend_irecv(ops):
                w.wait()                                   # (NCCL: enqueues on the current stream, does not block the host)
            if recv_slot is not None:
                self.eng.slot_end_access(recv_slot, self.comm.cuda_stream, True)
            if send_slot is not None:
                self.eng.slot_end_access(send_slot, self.comm.cuda_stream, False)
        self.bcast_bytes += self.slot_bytes * len(ops)
