"""The stage-1 -> stage-2 -> decode hand-off buffers of a session have three slots (step % 3), and the graphs that touch a slot and a
parity buffer have one copy per step % 6.  Stage 1 of step k then waits only for stage 2 and the decode slide of step k - 3, so it
runs beside the stage-2 forward of step k - 2.

Pipelining must not change a sample: the outputs of back-to-back device steps are bitwise equal to stepping one chunk at a time with
a device synchronise in between.  A guard that lets stage 1 or stage 2 overwrite a slot that an earlier step still reads, or a graph
copy that points at the wrong slot, shows up here as a difference.  Covered: one session at 0.1, 0.3 and 1.0 s chunks, a group of two,
and a member whose own step count differs from the group's in parity and modulo 3 when it joins (it ran 4 steps alone and joins at
group step 5).  Every run is 18 steps or more, so the 3- and 6-step cycles wrap several times.
"""
import numpy as np
import pytest

from realtime_yukarin_b200 import synthetic
from tests.test_gpu_analysis_chain import EXTRA, FS, _load

pytestmark = pytest.mark.gpu

STEPS = 18


def _cfg(T):
    from realtime_yukarin_b200.engine import SessionConfig
    return SessionConfig(fs=FS, frame_period_ms=5.0, f0_floor=71.0, f0_ceil=800.0, fft_length=1024, order=8, alpha=0.466, buffer_time=T,
                         encode_extra_time=EXTRA[0], convert_extra_time=EXTRA[1], decode_extra_time=EXTRA[2], threshold_db=60.0,
                         vocoder_buffer_size=1024)


def _run(engine, T, streams, plan, sync_each):
    """Run `plan` on fresh sessions 0..streams-1 from device memory and return every session's outputs in step order.

    plan items: ('alone', i) pushes one chunk to session i by itself; ('join', i) puts session i into the group (created at the first
    join); ('group',) pushes one chunk to every member.  Session i reads synthetic speech of stream 60 + i, chunk after chunk, and
    every step writes its own output slot.  sync_each: a device synchronise after every step, else all steps back to back."""
    import torch
    n = round(T * FS)
    sids = [engine.session_create(_cfg(T)) for _ in range(streams)]
    cap = engine.session_io_geometry(sids[0])['max_out']
    d_in = [torch.from_numpy(synthetic.synthetic_speech((len(plan) + 1) * T, stream=60 + i)[:len(plan) * n]).cuda() for i in range(streams)]
    d_out = torch.full((len(plan) * streams, cap), np.nan, dtype=torch.float64, device='cuda')
    d_n = torch.zeros(len(plan) * streams, dtype=torch.int32, device='cuda')
    torch.cuda.synchronize()
    steps, slots, members, gid = [0] * streams, [[] for _ in range(streams)], [], None

    def take(i):
        slot = sum(len(s) for s in slots)
        slots[i].append(slot)
        steps[i] += 1
        return d_in[i][(steps[i] - 1) * n:].data_ptr(), d_out[slot].data_ptr(), d_n[slot:].data_ptr()

    for item in plan:
        if item[0] == 'join':
            members.append(item[1])
            if gid is None:
                gid = engine.group_create([sids[item[1]]])
            else:
                engine.group_add(gid, sids[item[1]])
            continue
        if item[0] == 'alone':
            w, o, c = take(item[1])
            engine.session_push_device(sids[item[1]], w, n, o, cap, c)
        else:
            ptrs = [take(i) for i in members]
            engine.group_push_device(gid, [p[0] for p in ptrs], n, [p[1] for p in ptrs], cap, [p[2] for p in ptrs])
        if sync_each:
            engine.synchronize()
    engine.synchronize()
    torch.cuda.synchronize()
    outs, ns = d_out.cpu().numpy(), d_n.cpu().numpy()
    if gid is not None:
        engine.group_destroy(gid)
    for sid in sids:
        engine.session_destroy(sid)
    return [[outs[s, :ns[s]].copy() for s in slots[i]] for i in range(streams)]


def _check(engine, full_models, T, streams, plan):
    _load(engine, full_models)
    engine.set_precision('fp16')
    ref = _run(engine, T, streams, plan, sync_each=True)
    got = _run(engine, T, streams, plan, sync_each=False)
    for i in range(streams):
        assert len(ref[i]) >= STEPS, (i, len(ref[i]))
        produced = sum(len(o) for o in ref[i])
        assert produced > (len(ref[i]) - 6) * round(T * FS) // 2, (i, produced)     # the comparison covers real output
        for k, (a, b) in enumerate(zip(got[i], ref[i])):
            assert len(a) == len(b), (i, k, len(a), len(b))
            assert np.array_equal(a, b), (i, k, float(np.max(np.abs(a - b))) if len(a) else 0.0)


@pytest.mark.parametrize('T', [0.1, 0.3, 1.0])
def test_single_session_pipelined_equals_stepwise(engine, full_models, T):
    _check(engine, full_models, T, 1, [('alone', 0)] * STEPS)


def test_group_of_two_pipelined_equals_stepwise(engine, full_models):
    _check(engine, full_models, 0.3, 2, [('join', 0), ('join', 1)] + [('group',)] * STEPS)


def test_member_joining_at_odd_group_step_pipelined_equals_stepwise(engine, full_models):
    # session 1 joins with 4 steps of its own (parity 0, slot 1) at group step 5 (parity 1, slot 2)
    plan = [('alone', 1)] * 4 + [('join', 0)] + [('group',)] * 5 + [('join', 1)] + [('group',)] * (STEPS - 4)
    _check(engine, full_models, 0.3, 2, plan)
