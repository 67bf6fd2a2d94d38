"""N>1 path on CPU: the frame-parallel schedule (openhevc_b200/frame_parallel.py) with gloo, world_size 2.
Pictures are "decoded" by the test oracle; what is under test is the host logic the GPU path shares: ownership by intra
period, per-GPU DPB slot rotation, the deferred leading B pictures and the point-to-point exchange of the one anchor that
crosses GPUs.  Every picture must equal the sequential decode of the same stream."""
import hashlib
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import oracle_lib
from openhevc_b200 import frame_parallel as FP
from openhevc_b200 import worklist as W
from openhevc_b200.synth import FrameSynth, smooth_frame

W_, H_, CFI, BD = 128, 64, 1, 8


def make_small_blobs():
    blobs = []
    for i, (name, n_ref) in enumerate(FP.blob_specs()):
        blob, _ = FrameSynth(W_, H_, CFI, BD, seed=500 + i, refs=list(range(n_ref)), cur_slot=2, p_intra=0.1 if n_ref else 1.0).generate()
        blobs.append(blob)
    return blobs


class OracleBackend:
    def __init__(self, blobs, world):
        self.blobs, self.world = blobs, world
        self.dpb = [[np.zeros_like(p) for p in smooth_frame(W_, H_, CFI, BD, 0)] for _ in range(FP.N_SLOTS)]
        self.dpb[FP.anchor_slot(-1)] = smooth_frame(W_, H_, CFI, BD, 7)
        self.digests = {}
        self.n = 0
        self.g = 0

    def decode(self, pic, g=None):
        blob = self.blobs[pic.blob].copy()
        hdr = blob[:256].view(W.header_dt)
        hdr["cur_slot"] = pic.cur_slot
        hdr["n_ref"] = len(pic.ref_slots)
        hdr["ref_slot"][0][:len(pic.ref_slots)] = pic.ref_slots
        out = oracle_lib.execute(blob, self.dpb)
        self.dpb[pic.cur_slot] = [p.astype(np.uint8) for p in out]
        self.digests[(g, pic.blob)] = hashlib.md5(b"".join(p.tobytes() for p in self.dpb[pic.cur_slot])).hexdigest()

    def exchange_anchors(self, send_slot, dst, recv_slot, src):
        ops = []
        bufs = []
        if recv_slot is not None:
            bufs = [torch.from_numpy(p) for p in self.dpb[recv_slot]]
            ops += [dist.P2POp(dist.irecv, t, src) for t in bufs]
        if send_slot is not None:
            ops += [dist.P2POp(dist.isend, torch.from_numpy(p), dst) for p in self.dpb[send_slot]]
        if ops:
            for w in dist.batch_isend_irecv(ops):
                w.wait()


def worker(rank, world, port, k, q):
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    be = OracleBackend(make_small_blobs(), world)
    n = FP.run_schedule(be, rank, world, k)               # the product schedule itself (same call sequence as on GPUs)
    out = [None] * world
    dist.all_gather_object(out, (be.digests, n == len(be.digests)))
    if rank == 0:
        q.put(out)
    dist.destroy_process_group()


def test_two_rank_frame_parallel_equals_sequential():
    k = 8                                                 # GOPs per rank: two intra periods each
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=worker, args=(r, 2, port, k, q)) for r in range(2)]
    for p in procs:
        p.start()
    out = q.get(timeout=300)
    for p in procs:
        p.join(60)
        assert p.exitcode == 0
    par = {}
    for digests, same in out:
        assert same
        par.update(digests)
    # sequential reference: one rank decodes all 2k GOPs, in plain decode order
    seq = OracleBackend(make_small_blobs(), 1)
    for g in range(2 * k):
        for p in FP.gop_pictures(g):
            seq.decode(p, g)
    assert set(par) == set(seq.digests)
    bad = [key for key in seq.digests if seq.digests[key] != par[key]]
    assert not bad, bad


@pytest.mark.parametrize("n_gops", [1, 5, 8, 11])
def test_schedule_decodes_exactly_the_requested_gops(n_gops):
    """one rank: n_gops GOPs of 8 pictures, also when n_gops is no multiple of the intra period; every reference written first"""
    class Record:
        def __init__(self):
            self.pics, self.written = [], {FP.anchor_slot(-1)}

        def decode(self, pic, g=None):
            assert all(r in self.written for r in pic.ref_slots), (g, pic)
            self.written.add(pic.cur_slot)
            self.pics.append((g, pic))

        def exchange_anchors(self, *a):
            pass
    rec = Record()
    assert FP.run_schedule(rec, 0, 1, n_gops) == 8 * n_gops == len(rec.pics)
    assert sorted({g for g, _ in rec.pics}) == list(range(n_gops))


def test_schedule_with_several_ranks_decodes_a_prefix_of_the_stream():
    """two ranks, 5 GOPs asked: whole intra periods (8 GOPs per rank), GOPs 0..15 and nothing else"""
    class Record:
        def __init__(self):
            self.gops = set()

        def decode(self, pic, g=None):
            self.gops.add(g)

        def exchange_anchors(self, *a):
            pass
    recs = [Record(), Record()]
    assert [FP.run_schedule(r, rank, 2, 5) for rank, r in enumerate(recs)] == [64, 64]
    assert sorted(recs[0].gops | recs[1].gops) == list(range(16))


def test_gop_plan_is_consistent():
    for g in range(40):
        pics = FP.gop_pictures(g)
        assert len(pics) == 8 and pics[0].anchor and pics[0].cur_slot == g % FP.N_ANCHOR_SLOTS
        written = {FP.anchor_slot(g - 1)}
        for p in pics:
            assert all(r in written for r in p.ref_slots), (g, p)
            assert p.cur_slot not in p.ref_slots
            written.add(p.cur_slot)
    assert sum(1 for g in range(FP.INTRA_PERIOD_GOPS) if not FP.gop_pictures(g)[0].ref_slots) == 1
