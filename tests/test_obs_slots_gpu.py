"""The slot-ordered observation (magent_b200_get_observation_slots) on the GPU.

Every check compares the CUDA call with the CUDA row-ordered observation gathered through get_slots, bit for bit, with
vacant slots all +0.0 (tests/obs_slots_common.py): in every game mode and the fuzz configs, through host and device
pointers, into unaligned and over-long outputs, at battle512's full size after device restores, under forced render
launch shapes that make CTAs carry their tile across vacant and live records in every render instantiation, and
inside a replayed CUDA graph with a device restore."""
import ctypes
import itertools

import numpy as np
import pytest

import arena_restore_common as arc
import fuzz_common as fz
import obs_slots_common as oc
import parity_common as pc
import slots_common as sc

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]


def host_and_device(env, h, half):
    """the host-pointer call, after checking it bit for bit against the device-pointer call"""
    import torch
    rc, hv, hf = oc.call_host(env, h, half)
    assert rc == 0, env._lib.magent_b200_last_error()
    dv, df = env.get_observation_slots_torch(h, dtype=torch.float16 if half else torch.float32)
    u = np.uint16 if half else np.uint32
    assert np.array_equal(dv.cpu().numpy().view(u), hv.view(u)), "device and host pointers differ (views)"
    assert np.array_equal(df.cpu().numpy().view(u), hf.view(u)), "device and host pointers differ (features)"
    return hv, hf


@pytest.mark.parametrize("name", sorted(arc.SCENARIOS))
def test_cuda_equals_the_gathered_rows_in_every_game_mode(name):
    env = arc.SCENARIOS[name](pc.CUDA_LIB, 5, _num_arenas=3)
    tr = sc.Slots(env)
    tally = []
    sc.play_and_check(tr, 3, 3, oc.slots_reader(0, host_and_device, tally))
    sc.add_somewhere(tr, 1, seed=6)
    pool = tr.snapshot()
    sc.play_and_check(tr, 2, 4, oc.slots_reader(1, host_and_device, tally))
    tr.restore(pool, [2, -1, 1], src_kind="device")
    sc.play_and_check(tr, 2, 5, oc.slots_reader(0, host_and_device, tally))
    assert sum(tally) > 0


def test_cuda_under_fuzz_configs():
    tally = []
    for seed in (2, 5, 6, 8, 13, 14, 41, 1004, 70001, 70005, 100002):
        tr = sc.Slots(fz.make_env(pc.CUDA_LIB, seed, _num_arenas=4))
        sc.play_irregular(tr, 4, seed, oc.slots_reader(seed & 1, host_and_device, tally))
    assert sum(tally) > 0


def guarded(n_elems, half, offset):
    """a CUDA region of n_elems starting `offset` elements past a 16-byte boundary, with guard elements holding a NaN
    sentinel before it and 37 after it (an over-long output): (region, raw integers, guard before, sentinel)"""
    import torch
    guard = 16
    sentinel = 0x7da5 if half else 0x7fa5a5a5
    raw = torch.full((n_elems + guard + 37,), sentinel, dtype=torch.int16 if half else torch.int32, device="cuda")
    region = raw.view(torch.float16 if half else torch.float32)[guard - offset:guard - offset + n_elems]
    return region, raw, guard - offset, sentinel


@pytest.mark.parametrize("half", [0, 1], ids=["f32", "f16"])
def test_unaligned_and_over_long_outputs(half):
    """views and features one element past a 16-byte boundary (the render's element-store path) and aligned, inside
    longer buffers: equal to the restatement, nothing written outside the A * S records"""
    import torch
    env = pc.make_battle(pc.CUDA_LIB, 24, 50, 7, _num_arenas=3, _obs_launch=(2, 3, 0))
    tr = sc.Slots(env)
    env.select_arena(1)
    tr.add(tr.hs[0], method="random", n=9)
    env.select_arena(-1)
    rs = np.random.RandomState(1)
    for t in range(4):
        sc.random_step(env, rs, cull=t % 2 == 1)
        for g, h in enumerate(tr.hs):
            want_v, want_f, slot_row = oc.expected(env, h, half)
            for offset in (0, 1):
                vr, vraw, v0, sentinel = guarded(want_v.size, half, offset)
                fr, fraw, f0, _ = guarded(want_f.size, half, offset)
                bufs = (ctypes.c_void_p * 2)(vr.data_ptr(), fr.data_ptr())
                assert env._lib.magent_b200_get_observation_slots(env.game, g, bufs, half) == 0
                rep = env._get_obs_launch()
                assert rep["aligned"] == (1 - offset) and rep["tiles"] > rep["grid"], rep
                torch.cuda.synchronize()
                for raw, start, n in ((vraw, v0, want_v.size), (fraw, f0, want_f.size)):
                    edge = torch.cat([raw[:start], raw[start + n:]]).cpu().numpy()
                    assert (edge == sentinel).all(), "step %d group %d: a guard element was overwritten" % (t, g)
                oc.compare(vr.view(want_v.shape).cpu().numpy(), fr.view(want_f.shape).cpu().numpy(), want_v, want_f,
                           slot_row, half, "step %d group %d offset %d" % (t, g, offset))


def test_mixed_pointers_and_bad_outputs_are_refused():
    import torch
    env = pc.make_battle(pc.CUDA_LIB, 20, 37, 2, _num_arenas=3)
    h = env.get_handles()[1]
    g = env._hv(h)
    S = env.get_slot_space(h)
    vshape, fshape = (3, S) + env.view_space[g], (3, S) + env.feature_space[g]
    dv = torch.full(vshape, -9.0, device="cuda")
    df = torch.full(fshape, -9.0, device="cuda")
    hv = np.full(vshape, -9.0, np.float32)
    hf = np.full(fshape, -9.0, np.float32)
    L = env._lib
    for p in ((dv.data_ptr(), hf.ctypes.data), (hv.ctypes.data, df.data_ptr())):
        assert L.magent_b200_get_observation_slots(env.game, 1, (ctypes.c_void_p * 2)(*p), 0) == -1
        assert b"must both be host memory or both CUDA device memory" in L.magent_b200_last_error()
    torch.cuda.synchronize()
    assert (hv == -9).all() and (hf == -9).all() and bool((dv == -9).all()) and bool((df == -9).all())
    bad_outs = [
        (dv.cpu(), df),                                                         # host tensor
        (dv, df.half()),                                                        # mixed dtypes
        (dv.double(), df.double()),                                             # dtype
        (dv[:, :-1].contiguous(), df),                                          # not (A, S)
        (dv, torch.zeros((3, S) + (2 * fshape[2],), device="cuda")[..., ::2]),  # not contiguous
        dv,
    ]
    for bad in bad_outs:
        with pytest.raises(ValueError):
            env.get_observation_slots_torch(h, out=bad)
    with pytest.raises(ValueError):
        env.get_observation_slots_torch(h, dtype=torch.bfloat16)
    got_v, got_f = env.get_observation_slots_torch(h, out=(dv, df))
    oc.check(env, h, 0, lambda *_: (got_v.cpu().numpy(), got_f.cpu().numpy()))


def device_expected(env, h, half):
    """the restatement on the device: the row-ordered CUDA observation gathered through get_slots_torch"""
    import torch
    dt = torch.float16 if half else torch.float32
    rv, rf = env.get_observation_torch(h, dtype=dt)
    _rs, slot_row = env.get_slots_torch(h)
    idx = slot_row.clamp(min=0).long().view(-1)
    occ = (slot_row >= 0).view(slot_row.shape + (1,) * (rv.dim() - 1))
    it = torch.int16 if half else torch.int32
    zero = torch.zeros((), dtype=it, device="cuda")
    wv = torch.where(occ, rv.view(it)[idx].view(slot_row.shape + rv.shape[1:]), zero) if len(rv) else None
    wf = torch.where(occ[..., 0, 0, :], rf.view(it)[idx].view(slot_row.shape + rf.shape[1:]), zero) if len(rf) else None
    return wv, wf, slot_row


def test_battle512_at_full_size_after_device_restores():
    """bench.py's 512 arenas of 2 x 1000, device-resident steps with clear_dead and a tenth of the arenas restored from a
    device src every 4 steps: both groups, float32 and float16, against the gathered rows on the device"""
    import torch
    env = pc.make_battle(pc.CUDA_LIB, 200, 1000, 100, _num_arenas=512)
    hs = env.get_handles()
    A = 512
    pool = env.snapshot_arenas()
    rs = np.random.RandomState(3)
    done = torch.zeros((1,), dtype=torch.int32, device="cuda")
    vacant = 0
    for t in range(9):
        for g, h in enumerate(hs):
            env.set_random_legal_actions(h, 100 * t + g)
        env.step_device_done(done.data_ptr())
        env.clear_dead()
        if t % 4 == 3:
            src = np.full(A, -1, dtype=np.int32)
            pick = rs.choice(A, size=A // 10, replace=False)
            src[pick] = rs.randint(0, A, size=len(pick))
            env.restore_arenas(pool, torch.from_numpy(src).cuda())
        if t % 2 == 0 and t < 8:
            continue
        for g, h in enumerate(hs):
            half = (t + g) % 2
            it = torch.int16 if half else torch.int32
            gv, gf = env.get_observation_slots_torch(h, dtype=torch.float16 if half else torch.float32)
            wv, wf, slot_row = device_expected(env, h, half)
            what = "step %d group %d" % (t, g)
            assert torch.equal(gf.view(it), wf), what + ": features"
            assert torch.equal(gv.view(it), wv), what + ": views"
            vacant += int((slot_row < 0).sum())
            del gv, gf, wv, wf
    assert vacant > 0


# ---------------------------------------------------------------- forced launch shapes: vacant <-> live transitions
from test_render_reuse_gpu import COUNTS, SMEM_PER_BLOCK, VIEWS, make_config  # noqa: E402

FORCED_VIEWS = ("circle6", "circle8_nominimap", "circle10", "turn_sector")


def forced_cases():
    return list(itertools.product(FORCED_VIEWS, ("f32", "f16"), (1, 2)))


@pytest.mark.parametrize("view,dtype,tile", forced_cases(), ids=["%s-%s-tile%d" % c for c in forced_cases()])
def test_forced_launches_carry_the_tile_across_vacant_slots(view, dtype, tile):
    """small forced grids make every CTA render many tiles of the [A, S] records, so warps follow a vacant record with a
    live one and the other way round (a rebuild), and a vacant record with a vacant one (an undo).  Four arenas with
    ragged counts (an arena without group 0, one with a single agent, one without group 1: NaN minimap channels),
    culls after random steps and added agents scatter the vacant slots between live ones"""
    import magent_b200 as magent
    import torch
    half = dtype == "f16"
    esz = 2 if half else 4
    A = 4
    env = magent.GridWorld(make_config(view), _lib=pc.CUDA_LIB, _num_arenas=A, _obs_launch=(3, 2, tile))
    env.set_seed(22)
    env.reset()
    for a in range(A):
        env.select_arena(a)
        env.add_walls(method="random", n=40)
        for g, h in enumerate(env.get_handles()):
            if COUNTS[g][a]:
                env.add_agents(h, method="random", n=COUNTS[g][a])
    env.select_arena(-1)
    tr = sc.Slots(env)
    nit = 4 if view == "circle6" else 8
    turn = int(VIEWS[view][2])
    stats = {"undo_vacant": 0, "rebuild_vacancy": 0}
    rs = np.random.RandomState(5)
    for t in range(6):
        sc.random_step(env, rs, cull=t != 2)
        if t == 3:
            sc.add_somewhere(tr, 2, seed=t, n=5)
        for g, h in enumerate(tr.hs):
            gv, gf = env.get_observation_slots_torch(h, dtype=torch.float16 if half else torch.float32)
            rep = env._get_obs_launch()
            S = env.get_slot_space(h)
            what = "step %d group %d" % (t, g)
            oc.check(env, h, half, lambda *_: (gv.cpu().numpy(), gf.cpu().numpy()), what)
            if S == 0:
                continue
            vh, vw, C = env.view_space[g]
            lut = (4 if turn else 1) * ((vh * vw + 1) & ~1) * 8
            wide = tile == 2 and (32 // esz) * vh * vw * C * esz + lut <= SMEM_PER_BLOCK
            ta = (32 if wide else 16) // esz
            tiles = -(-A * S // ta)
            assert (rep["elem_bytes"], rep["nit"], rep["turn"], rep["tile_agents"], rep["tiles"]) == \
                (esz, nit, turn, ta, tiles), "%s: launch %s" % (what, rep)
            assert rep["grid"] == min(3, tiles) and tiles > rep["grid"], rep
            assert rep["chunk"] == 2, rep
            # the two tiles of a chunk go to one CTA one after the other, however the chunks are dealt: warp w follows
            # record o with record o + ta
            _r, slot_row = sc.read_host(env, h)
            vac = (slot_row < 0).reshape(-1)
            o1 = np.array([2 * c * ta + w for c in range(-(-tiles // 2)) for w in range(ta)])
            o1 = o1[o1 + ta < len(vac)]
            stats["undo_vacant"] += int((vac[o1] & vac[o1 + ta]).sum())
            stats["rebuild_vacancy"] += int((vac[o1] != vac[o1 + ta]).sum())
    assert stats["undo_vacant"] > 0 and stats["rebuild_vacancy"] > 0, stats


# ---------------------------------------------------------------- CUDA graphs
def test_restore_then_slot_observation_inside_a_replayed_cuda_graph():
    """two steps recorded with a restore of two arenas (a device src) and both groups' slot-ordered observations into
    fixed tensors (group 0 float32, group 1 float16), replayed 20 times with refilled actions, against an un-captured twin
    making the same calls with host buffers"""
    import torch
    from magent_b200.c_lib import load_library
    L = load_library(pc.CUDA_LIB)
    env, twin = (arc.make_duel(pc.CUDA_LIB, 3, _num_arenas=4) for _ in range(2))
    hs = env.get_handles()
    snap, tsnap = env.snapshot_arenas(), twin.snapshot_arenas()
    bound = [env.get_num_bound(h) for h in hs]
    na = env.get_action_space(hs[0])[0]
    dts = (torch.float32, torch.float16)
    acts = [[torch.zeros((n,), dtype=torch.int32, device="cuda") for n in bound] for _ in range(2)]
    outs = [[env.get_observation_slots_torch(hs[g], dtype=dts[g]) for g in range(2)] for _ in range(2)]
    done = torch.zeros((2,), dtype=torch.int32, device="cuda")
    src = np.array([1, -1, 3, -1], dtype=np.int32)
    d_src = torch.from_numpy(src).cuda()

    def one(k):
        for h, a in zip(hs, acts[k]):
            L.env_set_action(env.game, env._hv(h), a.data_ptr())
        env.step_device_done(done.data_ptr() + 4 * k)
        env.clear_dead()
        env.restore_arenas(snap, d_src)
        for g in range(2):
            env.get_observation_slots_torch(hs[g], out=outs[k][g])

    rs = np.random.RandomState(7)

    def draw():
        a = [[rs.randint(0, na, size=n).astype(np.int32) for n in bound] for _ in range(2)]
        for k in range(2):
            for g in range(2):
                acts[k][g].copy_(torch.from_numpy(a[k][g]))
        return a

    def twin_pair(a):
        out = []
        for k in range(2):
            ths = twin.get_handles()
            for h, x in zip(ths, a[k]):
                twin.set_action(h, np.ascontiguousarray(x[:twin.get_num(h)]))
            twin.step()
            twin.clear_dead()
            twin.restore_arenas(tsnap, src)
            out.append([oc.call_host(twin, ths[g], g)[1:] for g in range(2)])
        return out

    a = draw()
    one(0)
    one(1)
    twin_pair(a)
    for k in range(2):
        for g in range(2):
            for x in outs[k][g]:
                x.fill_(-3)
    gid = env.capture_graph(lambda: (one(0), one(1)))
    compared = 0
    for _ in range(20):
        a = draw()
        env.launch_graph(gid, 1)
        want = twin_pair(a)
        torch.cuda.synchronize()
        for k in range(2):
            for g, (wv, wf) in enumerate(want[k]):
                u = np.uint16 if g else np.uint32
                gv, gf = (x.cpu().numpy().view(u) for x in outs[k][g])
                assert np.array_equal(gv, wv.view(u)) and np.array_equal(gf, wf.view(u)), "replay, call %d group %d" % (k, g)
                compared += int((np.abs(wf).sum(-1) > 0).sum())
    assert compared > 0
