"""GPU: wire records (the format_results payload the assemble kernel emits), the hygiene fixes of round 2, and -- on a
box with >= 2 GPUs -- the NVLink gather (sharding.PeerWireSink: records stored straight into rank 0's buffer by the
assemble kernel) against a single-GPU run of the whole batch."""
import os
import socket

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def env(cuda_device):
    import torch
    from improved_body_parts_b200 import skeleton, synth, wire
    from improved_body_parts_b200.grouping import Grouper
    from oracle import spg_oracle as so

    class Env:
        pass

    e = Env()
    e.torch, e.skeleton, e.synth, e.wire, e.Grouper, e.so, e.dev = torch, skeleton, synth, wire, Grouper, so, cuda_device
    return e


def _group_with_wire(env, heat, paf, extent, params, rows=None, **cfg):
    t = env.torch
    N = heat.shape[0]
    g = env.Grouper(max_batch=N, max_h=heat.shape[2], max_w=heat.shape[3], **cfg)
    try:
        rows = g.capR if rows is None else rows
        buf = t.zeros((N + 2, g.wire_record_bytes(rows)), dtype=t.uint8, device=env.dev)
        g.set_wire_output(buf.data_ptr(), 1, rows)  # first_record = 1: record 0 and the last one must stay untouched
        g.group_device(t.from_numpy(heat).to(env.dev), t.from_numpy(paf).to(env.dev), extent, params)
        r = g.fetch()
        raw = buf.cpu().numpy()
        assert not raw[0].any() and not raw[-1].any()
        return r, env.wire.as_records(raw[1:-1], 17, rows)
    finally:
        g.close()


def test_wire_records_are_the_process_tail(env):
    """Records == people_xy / people_score of the same call == the checker's process() tail; the presence mask marks
    exactly the joints whose subset entry is not -1 (the reference's integer (0, 0) placeholder, evaluate.py:531)."""
    heat, paf = env.synth.make_batch(4242, 16, 128, 128, 18, drop_prob=0.2, edge=True)
    params = env.skeleton.default_params()
    r, rec = _group_with_wire(env, heat, paf, 128, params)
    o = env.so.group_batch(heat, paf, env.skeleton.LIMBS, 128, params, threads=4)
    assert (r.status == 0).all() and not rec["status"].any()
    assert np.array_equal(rec["n_persons"], r.n_persons) and np.array_equal(rec["n_persons"], o.n_persons)
    missing = 0
    for i in range(16):
        P = int(r.n_persons[i])
        xy, sc = o.to_coco(i, env.skeleton.COCO_FROM_PART)
        assert np.array_equal(rec[i]["rows"]["xy"][:P], xy) and np.array_equal(rec[i]["rows"]["score"][:P], sc)
        assert np.array_equal(rec[i]["rows"]["xy"][:P], r.people_xy[i, :P])
        ids = r.subset[i, :P][:, list(env.skeleton.COCO_FROM_PART), 0]
        want = ((ids >= 0) * (1 << np.arange(17))[None, :]).sum(axis=1).astype(np.uint64)
        assert np.array_equal(rec[i]["rows"]["present"][:P], want)
        missing += int((ids < 0).sum())
        assert not rec[i]["rows"]["xy"][P:].any()  # rows beyond n_persons are never written
    assert missing > 0
    people = env.wire.unpack(rec, list(range(16)))
    assert sum(len(v) for v in people.values()) == int(r.n_persons.sum())
    assert any(isinstance(x, int) for v in people.values() for pts, _ in v for x, _ in pts)


def test_armed_signal_is_published_by_the_assemble_kernel(env):
    """spg_arm_wire_signal: the last CTA of the next assemble launch release-stores the value (here into local memory);
    one shot -- the following launch leaves the word alone; both the fused and the stand-alone kernel carry it.  A
    multi-scale postnet at stride 2 between the two armed launches grows the handle's float64 accumulator, which must
    leave the signal's counter alone."""
    t = env.torch
    heat, paf = env.synth.make_batch(808, 9, 128, 128, 8)
    params = env.skeleton.default_params()
    g = env.Grouper(max_batch=9)
    try:
        hd, pd = t.from_numpy(heat).to(env.dev), t.from_numpy(paf).to(env.dev)
        buf = t.zeros((9, g.wire_record_bytes()), dtype=t.uint8, device=env.dev)
        word = t.zeros((2,), dtype=t.int64, device=env.dev)
        g.set_wire_output(buf.data_ptr())
        g.arm_wire_signal(word.data_ptr(), 41)
        g.group_device(hd, pd, 128, params)            # fused match_assemble
        t.cuda.synchronize()
        assert word.tolist() == [41, 0]
        first = buf.cpu().numpy()
        gen = t.Generator().manual_seed(5)
        net = [t.rand((1, 2, 50, 40, 48), generator=gen).to(env.dev) for _ in range(2)]
        g.postnet(net, [(76, 90), (70, 84)], (61, 77), stride=2, paf_dtype=t.float64)
        g.group_device(hd, pd, 128, params)            # not armed any more
        g.arm_wire_signal(word.data_ptr() + 8, 77)
        g.assemble(9, params)                          # the stand-alone kernel
        t.cuda.synchronize()
        assert word.tolist() == [41, 77]
        assert np.array_equal(buf.cpu().numpy(), first)
        rec = env.wire.as_records(buf.cpu().numpy(), 17, g.capR)
        assert (rec["n_persons"] > 0).all()
        g.set_wire_output(None)
        from improved_body_parts_b200.grouping import GroupingError
        with pytest.raises(GroupingError, match="wire output"):
            g.arm_wire_signal(word.data_ptr(), 1)
    finally:
        g.close()


def test_wire_row_capacity_is_flagged_not_overrun(env):
    from improved_body_parts_b200.grouping import ST_WIRE_OVERFLOW
    heat, paf = env.synth.make_batch(77, 3, 96, 96, 6)
    params = env.skeleton.default_params()
    r, rec = _group_with_wire(env, heat, paf, 96, params, rows=2)
    assert (r.n_persons > 2).all()
    assert (rec["n_persons"] == 2).all() and (rec["status"] & ST_WIRE_OVERFLOW).all() and (r.status & ST_WIRE_OVERFLOW).all()
    for i in range(3):
        assert np.array_equal(rec[i]["rows"]["xy"], r.people_xy[i, :2])


@pytest.mark.parametrize("mid_num", [64, 65, 100])
@pytest.mark.parametrize("H,scale,persons", [(128, (5.0, 5.6), 3), (160, (5.5, 6.5), 4)])
def test_mid_num_beyond_the_reciprocal_table(env, mid_num, H, scale, persons):
    """ADVICE r1: mid_num > 64 used to read past the per-m reciprocal table.  The reference accepts any mid_num (the
    checker agrees with the live reference at mid_num 65 / 100 on these inputs, bit for bit).  128x128 takes the
    persistent kernel, 160x160 the per-item one; both have accepted limbs longer than 64 px."""
    from test_gpu_parity import _assert_same
    heat, paf = env.synth.make_batch(606, 4, H, H, persons, scale_range=scale, sigma_scale=3.0)
    params = dict(env.skeleton.default_params(), mid_num=mid_num)
    o = env.so.group_batch(heat, paf, env.skeleton.LIMBS, H, params)
    r, _ = _group_with_wire(env, heat, paf, H, params)
    assert (r.status == 0).all() and (o.status == 0).all() and r.n_persons.sum() > 0
    live = np.arange(r.conn_norm.shape[2])[None, None, :] < r.conn_count.clip(0)[:, :, None]
    assert (r.conn_norm[live] > 66).sum() > 20, "accepted limbs must be long enough to take more than 64 samples"
    for i in range(4):
        _assert_same(o.as_reference_structures(i), r.as_reference_structures(i), f"mid_num={mid_num} image {i}")


def test_debug_environment_cannot_change_results(env, monkeypatch):
    """VERDICT r1 weak #7: SPG_DEBUG_PERSIST used to switch the scorer off in the production library."""
    heat, paf = env.synth.make_batch(99, 8, 128, 128, 20)
    params = env.skeleton.default_params()
    a, _ = _group_with_wire(env, heat, paf, 128, params)
    monkeypatch.setenv("SPG_DEBUG_PERSIST", "1")
    b, _ = _group_with_wire(env, heat, paf, 128, params)
    monkeypatch.setenv("SPG_DEBUG_PERSIST", "2")
    c, _ = _group_with_wire(env, heat, paf, 128, params)
    for f in ("conn_count", "cand_count", "n_persons", "subset", "people_xy"):
        assert np.array_equal(getattr(a, f), getattr(b, f)) and np.array_equal(getattr(a, f), getattr(c, f)), f
    assert a.n_persons.sum() > 100


def test_fused_match_assemble_equals_the_two_kernels(env, monkeypatch):
    """spg_group_batch runs limb_match + assemble fused in one kernel (matcher warps feed the assembler warp through
    shared memory); SPG_FUSE_MA=0 runs the two kernels back to back.  Same tables, same persons, same wire records --
    on clean and dirty crowds (merge / replace / overlap branches, > 32 connections per limb, special_k limbs)."""
    for seed, P, kw in ((31, 30, {}), (32, 40, dict(drop_prob=0.15, stretch=10, spikes=40, plateau=4, colocate=5, edge=True)),
                        (33, 10, dict(missing_parts=(4, 16), drop_prob=0.3))):
        heat, paf = env.synth.make_batch(seed, 12, 128, 128, P, **kw)
        params = dict(env.skeleton.default_params(), remove_recon=seed % 2)
        monkeypatch.setenv("SPG_FUSE_MA", "1")
        a, ra = _group_with_wire(env, heat, paf, 128, params, max_person_rows=128, max_peaks_per_part=128)
        monkeypatch.setenv("SPG_FUSE_MA", "0")
        b, rb = _group_with_wire(env, heat, paf, 128, params, max_person_rows=128, max_peaks_per_part=128)
        assert (a.status == 0).all() and (b.status == 0).all()
        live = np.arange(a.conn_ij.shape[2])[None, None, :] < a.conn_count.clip(0)[:, :, None]
        for f in ("conn_count", "n_persons", "subset", "people_xy", "people_score"):
            assert np.array_equal(getattr(a, f), getattr(b, f)), f
        for f in ("conn_ij", "conn_score", "conn_norm"):
            assert np.array_equal(getattr(a, f)[live], getattr(b, f)[live]), f
        assert ra.tobytes() == rb.tobytes()
        o = env.so.group_batch(heat, paf, env.skeleton.LIMBS, 128, params, threads=4)
        from test_gpu_parity import _assert_same
        for i in range(12):
            _assert_same(o.as_reference_structures(i), a.as_reference_structures(i), f"seed {seed} image {i}")


def test_stage_entry_points_validate_their_inputs(env):
    """ADVICE r1: nms_peaks / limb_score skipped the dtype / channel / shape checks of group_device."""
    from improved_body_parts_b200.grouping import GroupingError
    t = env.torch
    g = env.Grouper(max_batch=2)
    try:
        heat = t.zeros((2, 18, 128, 128), device=env.dev)
        with pytest.raises(GroupingError, match="float32"):
            g.nms_peaks(heat.double())
        with pytest.raises(GroupingError, match="channels"):
            g.nms_peaks(heat[:, :10])
        with pytest.raises(GroupingError, match="images"):
            g.nms_peaks(t.zeros((3, 18, 128, 128), device=env.dev))
        g.nms_peaks(heat)
        with pytest.raises(GroupingError, match="channels"):
            g.limb_score(t.zeros((2, 12, 128, 128), device=env.dev), 128)
        with pytest.raises(GroupingError, match="peaks on the device"):
            g.limb_score(t.zeros((2, 30, 64, 128), device=env.dev), 128)
        with pytest.raises(GroupingError, match="float32 or float64"):
            g.limb_score(t.zeros((2, 30, 128, 128), device=env.dev, dtype=t.float16), 128)
    finally:
        g.close()


# ---- two GPUs: the NVLink gather ---------------------------------------------------------------------------------
def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _peer_worker(rank, world, port, n_images, mode, q):
    import torch
    import torch.distributed as dist

    from improved_body_parts_b200 import skeleton, synth, wire
    from improved_body_parts_b200.grouping import Grouper
    from improved_body_parts_b200.sharding import PackedGather, PeerWireSink, shard_range

    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    armed = mode == "peer-armed"  # the assemble kernel's last CTA publishes the step itself (spg_arm_wire_signal)
    mode = "peer" if armed else mode
    dist.init_process_group("nccl" if mode == "packed" else "gloo", rank=rank, world_size=world,
                            **({"device_id": dev} if mode == "packed" else {}))
    try:
        lo, hi = shard_range(n_images, rank, world)
        params = skeleton.default_params()
        ROWS = 48
        g = Grouper(max_batch=max(hi - lo, 1), max_person_rows=64, device=rank)
        rb = g.wire_record_bytes(ROWS)
        stream = torch.cuda.current_stream()
        landed = None
        if mode == "peer":
            sink = PeerWireSink(hi - lo, rb, rank, dst=0, slots=2)
            cstream = torch.cuda.Stream(device=dev) if rank == 0 else None
        else:
            pg = PackedGather(hi - lo, rb, dev, dst=0)
        for s in range(5):  # different images every pass: a stale generation would be noticed
            heat, paf = synth.make_batch(9000 + 1000 * s + lo, hi - lo, 128, 128, 12)
            hd, pd = torch.from_numpy(heat).to(dev), torch.from_numpy(paf).to(dev)
            if mode == "peer":
                g.set_wire_output(sink.begin(s, stream), 0, ROWS)
                if armed:
                    g.arm_wire_signal(sink.counter_address(s), s + 1)
            else:
                g.set_wire_output(pg.local.data_ptr(), 0, ROWS)
            g.group_device(hd, pd, 128, params)
            if mode == "peer":
                if not armed:
                    sink.publish(s, stream)
                if rank == 0:
                    view = sink.collect(s, cstream)
                    with torch.cuda.stream(cstream):
                        landed = view.clone()  # consume, then hand the generation back
                    sink.release(s, cstream)
            else:
                pg.gather()
                if rank == 0:
                    landed = pg.records().clone()
        torch.cuda.synchronize()
        if rank == 0:
            q.put(landed.cpu().numpy())
        else:
            q.put("ok")
        dist.barrier()
        if mode == "peer":
            sink.close()
        g.close()
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("mode,n", [("peer", 12), ("peer", 7), ("peer-armed", 12), ("peer-armed", 5), ("packed", 7)])
def test_two_gpu_gather_equals_one_gpu(env, mode, n):
    t = env.torch
    if t.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp

    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_peer_worker, args=(r, 2, port, n, mode, q)) for r in range(2)]
    for p in procs:
        p.start()
    results = [q.get(timeout=300) for _ in procs]
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    got = env.wire.as_records(next(r for r in results if not isinstance(r, str)), 17, 48)
    # one GPU, whole batch, last pass's images (seeds are per image, so the shards are slices of this batch)
    heat, paf = env.synth.make_batch(9000 + 4000, n, 128, 128, 12)
    r, rec = _group_with_wire(env, heat, paf, 128, env.skeleton.default_params(), rows=48)
    assert len(got) == n and np.array_equal(got["n_persons"], rec["n_persons"]) and rec["n_persons"].sum() > 0
    assert not got["status"].any()
    # rows beyond n_persons are never written, so a slot keeps what an earlier pass (other images) left there: compare
    # the live part of every record, byte for byte
    for i in range(n):
        P = int(rec[i]["n_persons"])
        assert got[i]["rows"][:P].tobytes() == rec[i]["rows"][:P].tobytes(), f"image {i}"
