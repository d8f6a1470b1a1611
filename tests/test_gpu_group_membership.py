"""Sessions joining and leaving a running group between steps (ryk_group_add / _remove / _members).

  * membership is invisible in the audio: streams that join (at a step parity that differs from the group's, and one that matches), leave
    and rejoin have the per-step lengths of their voice's oracle stream and match it to the headline tolerance;
  * leaving is bitwise the ungroup path of ryk_group_destroy; removing member 0 is bitwise destroying the group and creating one of the
    remaining running sessions, and launches as many kernels afterwards; a joiner's output does not depend on its partner, through
    submit / collect and through push_device; the change calls launch nothing;
  * refused changes fail with their message, launch nothing and leave the member list as it was; a voice held by a member cannot go;
    add / remove cycles return their device memory; a re-blocker attached to a session that joins and leaves matches the host re-blocker.

The voices are created on the shared engine from their own seeded model files and destroyed at the end, with every session and group.
"""
import numpy as np
import pytest

from oracle import nets as onets
from oracle import pipeline as opipe
from realtime_yukarin_b200 import synthetic

pytestmark = pytest.mark.gpu

CFG = opipe.PathConfig()
TOL = 1e-3                  # headline tolerance: sample RMSE
T, FS = 0.3, 24000
N = round(T * FS)
DEPTH = 4                   # chunks in flight through submit / collect
STEPS = 12                  # chunks of every input stream


def _cfg(extra=(0.0, 0.5, 0.0), T=T):
    from realtime_yukarin_b200.engine import SessionConfig
    return SessionConfig(fs=FS, frame_period_ms=5.0, f0_floor=71.0, f0_ceil=800.0, fft_length=1024, order=8, alpha=0.466,
                         buffer_time=T, encode_extra_time=extra[0], convert_extra_time=extra[1], decode_extra_time=extra[2],
                         threshold_db=60.0, vocoder_buffer_size=1024)


def _rmse(a, b):
    return float(np.sqrt(np.mean((np.asarray(a, np.float64) - np.asarray(b, np.float64)) ** 2)))


def _speech(stream):
    return synthetic.synthetic_speech((STEPS + 1) * T, stream=stream)


def _load_voice(engine, paths):
    from realtime_yukarin_b200.models import load_voice
    v = engine.voice_create()
    load_voice(engine, v, **{k: paths[k] for k in ('stage1_model_path', 'stage2_model_path', 'input_statistics_path',
                                                     'target_statistics_path')})
    return v


@pytest.fixture(scope='module')
def voice_files(tmp_path_factory):
    """Two base-64 voices (seeds 31, 32) and a base-16 one (seed 33), none shared with the other test modules."""
    out = {seed: synthetic.write_synthetic_models(tmp_path_factory.mktemp(f'member{seed}'), seed=seed) for seed in (31, 32)}
    out[33] = synthetic.write_synthetic_models(tmp_path_factory.mktemp('member33'), seed=33, base1=16, base2=16)
    return out


@pytest.fixture(scope='module')
def voices(engine, voice_files):
    """[v1, v2]: the two base-64 voices loaded on the shared engine; destroyed afterwards."""
    engine.set_precision('fp16')
    ids = [_load_voice(engine, voice_files[seed]) for seed in (31, 32)]
    yield ids
    for v in ids:
        engine.voice_destroy(v)


_ORACLE = {}


def _oracle(paths, stream):
    """Per-step outputs of the oracle stream of `paths` over the STEPS chunks of _speech(stream) (a stream's first k outputs are those
    of its first k chunks)."""
    key = (str(paths['stage2_model_path']), stream)
    if key not in _ORACLE:
        from realtime_yukarin_b200.models import F0Converter
        f0c = F0Converter(paths['input_statistics_path'], paths['target_statistics_path'])
        p1, p2 = onets.load_npz(paths['stage1_model_path']), onets.load_npz(paths['stage2_model_path'])
        orc = opipe.StreamOracle(CFG, p1, p2, f0c.stats(), buffer_time=T, extra=(0.0, 0.5, 0.0), backend='torch')
        x = _speech(stream)
        _ORACLE[key] = [orc.push(x[k * N:(k + 1) * N]) for k in range(STEPS)]
    return _ORACLE[key]


class _Made:
    """Everything a test creates on the shared engine, destroyed in close() whatever failed."""

    def __init__(self, engine):
        self.engine, self.groups, self.sessions, self.reblocks, self.voices = engine, [], [], [], []

    def session(self, voice, cfg=None):
        self.sessions.append(self.engine.session_create(cfg or _cfg(), voice=voice))
        return self.sessions[-1]

    def group(self, sids):
        self.groups.append(self.engine.group_create(sids))
        return self.groups[-1]

    def close(self):
        e = self.engine
        e.set_precision('fp16')
        for items, destroy in ((self.groups, e.group_destroy), (self.reblocks, e.reblock_destroy), (self.sessions, e.session_destroy),
                               (self.voices, e.voice_destroy)):
            while items:
                destroy(items.pop())


@pytest.fixture
def made(engine):
    m = _Made(engine)
    yield m
    m.close()


class _Streams:
    """Sessions fed their own input streams, stepped alone or in groups.  Host mode: submit / collect with up to DEPTH chunks in
    flight per session or group; device mode: session_push_device / group_push_device, one step at a time.  outs[sid] = per-step
    outputs of session sid in step order, wherever each step ran.  A session with a re-blocker attached gets one device push behind
    each of its steps, its results in rb[sid].  change() collects everything before a membership change."""

    def __init__(self, engine, device=False):
        self.e, self.device = engine, device
        self.x, self.next, self.outs, self.queues, self.rid, self.rb = {}, {}, {}, {}, {}, {}

    def add(self, sid, x):
        self.x[sid], self.next[sid], self.outs[sid], self.rb[sid] = x, 0, [], []
        return sid

    def attach(self, sid, rid):
        self.rid[sid] = rid

    def _chunk(self, sid):
        k = self.next[sid]
        self.next[sid] += 1
        return self.x[sid][k * N:(k + 1) * N]

    def alone(self, sid):
        self._step(('s', sid), [sid])

    def group(self, gid):
        self._step(('g', gid), self.e.group_members(gid))

    def _step(self, key, sids):
        e = self.e
        chunks = [self._chunk(s) for s in sids]
        if self.device:
            self._step_device(key, sids, chunks)
            return
        t = e.session_submit(key[1], chunks[0]) if key[0] == 's' else e.group_submit(key[1], chunks)
        rts = {s: e.reblock_push_device(self.rid[s], session_id=s) for s in sids if s in self.rid}
        q = self.queues.setdefault(key, [])
        q.append((t, sids, rts))
        if len(q) >= DEPTH:
            self._collect(key)

    def _step_device(self, key, sids, chunks):
        import torch
        e = self.e
        dev = torch.device('cuda', e.device)
        cap = max(e.session_io_geometry(s)['max_out'] for s in sids)
        ws = [torch.from_numpy(np.ascontiguousarray(c, np.float32)).to(dev) for c in chunks]
        outs = [torch.zeros(cap, dtype=torch.float64, device=dev) for _ in sids]
        ns = [torch.zeros(1, dtype=torch.int32, device=dev) for _ in sids]
        torch.cuda.synchronize(dev)
        if key[0] == 's':
            e.session_push_device(key[1], ws[0].data_ptr(), N, outs[0].data_ptr(), cap, ns[0].data_ptr())
        else:
            e.group_push_device(key[1], [w.data_ptr() for w in ws], N, [o.data_ptr() for o in outs], cap, [c.data_ptr() for c in ns])
        e.synchronize()
        for s, o, c in zip(sids, outs, ns):
            self.outs[s].append(o[:int(c.item())].cpu().numpy().copy())

    def _collect(self, key):
        e = self.e
        t, sids, rts = self.queues[key].pop(0)
        bufs = [np.empty(65536) for _ in sids]
        got = [e.session_collect(key[1], t, bufs[0])] if key[0] == 's' else e.group_collect(key[1], t, bufs)
        for s, o in zip(sids, got):
            self.outs[s].append(o.copy())
        for s, rt in rts.items():
            st, chunk, power = e.reblock_collect(self.rid[s], rt)
            self.rb[s].append((st, None if chunk is None else chunk.copy(), power))

    def drain(self):
        for key in list(self.queues):
            while self.queues[key]:
                self._collect(key)

    def change(self, call):
        self.drain()
        call()


def _check_oracle(outs, paths, stream, what):
    refs = _oracle(paths, stream)[:len(outs)]
    assert [len(o) for o in outs] == [len(r) for r in refs], what
    err = _rmse(np.concatenate(outs), np.concatenate(refs))
    print(f'{what}: {len(outs)} steps, rmse {err:.3e}')
    assert err <= TOL, what


def test_join_leave_rejoin_match_the_oracle(engine, voices, voice_files, made):
    v1, v2 = voices
    files = {v1: voice_files[31], v2: voice_files[32]}
    # scenario 1: A runs alone for 3 steps and joins {P} at group step 4 (its own step 3: the other parity), B runs alone for 4 steps and
    # joins at group step 4 too (same parity); A leaves at group step 9 and runs alone to the end.  P runs the whole time.
    run = _Streams(engine)
    src = {}
    a, b, p = (run.add(made.session(v), _speech(s)) for v, s in ((v1, 401), (v1, 402), (v2, 403)))
    src.update({a: (v1, 401), b: (v1, 402), p: (v2, 403)})
    gid = made.group([p])
    for t in range(STEPS):
        if t == 4:
            run.change(lambda: (engine.group_add(gid, a), engine.group_add(gid, b)))
            assert engine.group_members(gid) == [p, a, b]
        if t == 9:
            run.change(lambda: engine.group_remove(gid, a))
            assert engine.group_members(gid) == [p, b]
        run.group(gid)
        if t < 3 or t >= 9:
            run.alone(a)
        if t < 4:
            run.alone(b)
    run.drain()
    assert [len(run.outs[s]) for s in (a, b, p)] == [3 + 5 + 3, STEPS, STEPS]
    # scenario 2: {X, Y, Z}; the middle one leaves at step 5, runs alone, and comes back (as the last member) at step 8
    run2 = _Streams(engine)
    x, y, z = (run2.add(made.session(v), _speech(s)) for v, s in ((v1, 401), (v2, 403), (v1, 402)))
    src.update({x: (v1, 401), y: (v2, 403), z: (v1, 402)})
    gid2 = made.group([x, y, z])
    for t in range(STEPS - 1):
        if t == 5:
            run2.change(lambda: engine.group_remove(gid2, y))
            assert engine.group_members(gid2) == [x, z]
        if t == 8:
            run2.change(lambda: engine.group_add(gid2, y))
            assert engine.group_members(gid2) == [x, z, y]
        run2.group(gid2)
        if 5 <= t < 8:
            run2.alone(y)
    run2.drain()
    for r, sids in ((run, (a, b, p)), (run2, (x, y, z))):
        for s in sids:
            v, stream = src[s]
            _check_oracle(r.outs[s], files[v], stream, f'session {s} (voice {v}, stream {stream})')


def _leave_run(engine, made, voices, destroy, j=5, after=4):
    """{A, P} for j steps, then A leaves (group_remove, or group_destroy ungrouping both) and runs `after` steps alone."""
    v1, _ = voices
    run = _Streams(engine)
    a, p = (run.add(made.session(v1), _speech(s)) for s in (411, 412))
    gid = made.group([a, p])
    for _ in range(j):
        run.group(gid)
    if destroy:
        run.change(lambda: engine.group_destroy(gid))
        made.groups.remove(gid)
    else:
        before = engine.launch_count
        run.change(lambda: engine.group_remove(gid, a))
        assert engine.launch_count == before
        assert engine.group_members(gid) == [p]
    for _ in range(after):
        run.alone(a)
    run.drain()
    return run.outs[a]


def test_leaving_is_bitwise_the_ungroup_path(engine, voices, made):
    j = 5
    removed = _leave_run(engine, made, voices, destroy=False, j=j)
    ungrouped = _leave_run(engine, made, voices, destroy=True, j=j)
    assert len(removed) == len(ungrouped) == j + 4
    for k in range(j, len(removed)):
        assert np.array_equal(removed[k], ungrouped[k]), k


def _compaction_run(engine, made, voices, recreate, j=4, after=5):
    """{A, B, C} (A on the other voice, so the plan moves to another net) for j steps, then A goes (group_remove, or group_destroy
    and group_create([B, C]) of the running sessions); `after` steps of the group of B and C.  Returns (outputs, launches after)."""
    v1, v2 = voices
    run = _Streams(engine)
    a, b, c = (run.add(made.session(v), _speech(s)) for v, s in ((v2, 421), (v1, 422), (v1, 423)))
    gid = made.group([a, b, c])
    for _ in range(j):
        run.group(gid)
    if recreate:
        def swap():
            engine.group_destroy(gid)
            made.groups.remove(gid)
            return made.group([b, c])
        run.drain()
        gid = swap()
    else:
        before = engine.launch_count
        run.change(lambda: engine.group_remove(gid, a))
        assert engine.launch_count == before
    assert engine.group_members(gid) == [b, c]
    before = engine.launch_count
    for _ in range(after):
        run.group(gid)
    run.drain()
    return run.outs, engine.launch_count - before, (b, c)


def test_compaction_is_bitwise_a_recreated_group(engine, voices, made):
    j = 4
    removed, removed_launches, (b1, c1) = _compaction_run(engine, made, voices, recreate=False, j=j)
    recreated, recreated_launches, (b2, c2) = _compaction_run(engine, made, voices, recreate=True, j=j)
    print(f'launches of 5 steps after the change: {removed_launches} (removed), {recreated_launches} (recreated)')
    assert removed_launches == recreated_launches
    for s1, s2 in ((b1, b2), (c1, c2)):
        assert len(removed[s1]) == len(recreated[s2]) == j + 5
        for k in range(j, j + 5):
            assert np.array_equal(removed[s1][k], recreated[s2][k]), (s1, k)


def _join_run(engine, made, voices, partner_voice, partner_stream, device, j=5, after=4):
    """A runs alone for j steps and joins the running {partner} at its step j; `after` group steps.  Returns A's outputs."""
    run = _Streams(engine, device=device)
    a = run.add(made.session(voices[0]), _speech(431))
    q = run.add(made.session(partner_voice), _speech(partner_stream))
    gid = made.group([q])
    for _ in range(j):
        run.alone(a)
        run.group(gid)
    before = engine.launch_count
    run.change(lambda: engine.group_add(gid, a))
    assert engine.launch_count == before
    assert engine.group_members(gid) == [q, a]
    for _ in range(after):
        run.group(gid)
    run.drain()
    return run.outs[a]


def test_joiner_does_not_depend_on_its_partner(engine, voices, made):
    v1, v2 = voices
    j = 5
    with_p = _join_run(engine, made, voices, v1, 432, device=False, j=j)
    with_q = _join_run(engine, made, voices, v2, 433, device=False, j=j)
    with_p_dev = _join_run(engine, made, voices, v1, 432, device=True, j=j)
    with_q_dev = _join_run(engine, made, voices, v2, 433, device=True, j=j)
    for k in range(len(with_p)):
        assert np.array_equal(with_p_dev[k], with_p[k]), k
        assert np.array_equal(with_q_dev[k], with_q[k]), k
    for k in range(j, len(with_p)):
        assert np.array_equal(with_p[k], with_q[k]), k
        assert np.array_equal(with_p_dev[k], with_q_dev[k]), k


def _refused(engine, call, needle, gid, members):
    from realtime_yukarin_b200.engine import RykError
    before = engine.launch_count
    with pytest.raises(RykError, match=needle):
        call()
    assert engine.launch_count == before
    assert engine.group_members(gid) == members


def test_refused_changes_leave_the_group_as_it_was(engine, voices, voice_files, made):
    v1, v2 = voices
    run = _Streams(engine)
    p = run.add(made.session(v2), _speech(403))
    gid = made.group([p])
    run.group(gid)
    run.drain()
    a = run.add(made.session(v1), _speech(401))
    # an uncollected ticket on the group, then on the session
    t = engine.group_submit(gid, [run._chunk(p)])
    _refused(engine, lambda: engine.group_add(gid, a), 'collect every submitted chunk of the group', gid, [p])
    run.outs[p].append(engine.group_collect(gid, t, [np.empty(65536)])[0].copy())
    t = engine.session_submit(a, run._chunk(a))
    _refused(engine, lambda: engine.group_add(gid, a), 'collect every submitted chunk of a session', gid, [p])
    run.outs[a].append(engine.session_collect(a, t, np.empty(65536)).copy())
    # a session already in a group
    other = made.session(v1)
    made.group([other])
    _refused(engine, lambda: engine.group_add(gid, other), 'already in a group', gid, [p])
    # another window length / chunk length and device rate
    shorter = made.session(v2, _cfg(extra=(0.0, 0.25, 0.0)))
    _refused(engine, lambda: engine.group_add(gid, shorter), 'same window length', gid, [p])
    rated = made.session(v2)
    engine.session_set_input_rate(rated, 48000)
    _refused(engine, lambda: engine.group_add(gid, rated), 'same device input and output rates', gid, [p])
    # a base-16 voice into a base-64 group
    made.voices.append(_load_voice(engine, voice_files[33]))
    narrow = made.session(made.voices[-1])
    _refused(engine, lambda: engine.group_add(gid, narrow), 'same', gid, [p])
    # a 9th voice: a group of 8 distinct base-64 voices takes no member of another voice
    extra = [v1, v2]
    for _ in range(7):
        made.voices.append(_load_voice(engine, voice_files[31]))
        extra.append(made.voices[-1])
    eight = made.group([made.session(v) for v in extra[:8]])
    members8 = engine.group_members(eight)
    ninth = made.session(extra[8])
    _refused(engine, lambda: engine.group_add(eight, ninth), 'at most 8', eight, members8)
    # a second voice in precision 0
    engine.set_precision('fp32')
    try:
        _refused(engine, lambda: engine.group_add(gid, a), 'precision', gid, [p])
    finally:
        engine.set_precision('fp16')
    # removing a non-member, removing the last member
    _refused(engine, lambda: engine.group_remove(gid, a), 'not a member', gid, [p])
    _refused(engine, lambda: engine.group_remove(gid, p), 'last member', gid, [p])
    # the group still steps, and so does A, which joins it now
    engine.group_add(gid, a)
    for _ in range(4):
        run.group(gid)
    run.drain()
    _check_oracle(run.outs[p], voice_files[32], 403, f'session {p} after the refusals')
    _check_oracle(run.outs[a], voice_files[31], 401, f'session {a} after the refusals')


def test_a_members_voice_cannot_go(engine, voices, voice_files, made):
    from realtime_yukarin_b200.engine import RykError
    run = _Streams(engine)
    p = run.add(made.session(voices[0]), _speech(403))
    gid = made.group([p])
    v = _load_voice(engine, voice_files[32])
    made.voices.append(v)
    s = run.add(made.session(v), _speech(404))
    run.alone(s)
    run.change(lambda: engine.group_add(gid, s))
    run.group(gid)
    run.drain()
    with pytest.raises(RykError, match='in use'):
        engine.voice_destroy(v)
    engine.group_remove(gid, s)
    with pytest.raises(RykError, match='in use'):
        engine.voice_destroy(v)
    made.sessions.remove(s)
    engine.session_destroy(s)
    made.voices.remove(v)
    engine.voice_destroy(v)


def test_membership_cycles_return_device_memory(engine, voices, made):
    import torch
    v1, v2 = voices
    run = _Streams(engine)
    p = run.add(made.session(v1), _speech(441))
    others = [run.add(made.session(v), _speech(442 + i)) for i, v in enumerate((v2, v1, v2))]
    gid = made.group([p])
    free = {}
    for cycle in range(1, 7):
        for s in others:                          # up to B = 4
            run.change(lambda: engine.group_add(gid, s))
            run.group(gid)
        for s in others:
            run.change(lambda: engine.group_remove(gid, s))
            run.alone(s)
        run.group(gid)
        run.drain()
        for s in others:                          # the streams restart every cycle: only the membership changes matter here
            run.next[s] = 0
        run.next[p] = 0
        if cycle in (2, 6):
            engine.synchronize()
            free[cycle] = torch.cuda.mem_get_info()[0]
    grown = (free[2] - free[6]) / 2**20
    print(f'device memory in use grew by {grown:.1f} MiB over 4 add / remove cycles')
    assert abs(grown) < 4.0


def test_reblocker_follows_a_session_that_joins_and_leaves(engine, voices, made):
    v1, v2 = voices
    run = _Streams(engine)
    a = run.add(made.session(v1), _speech(451))
    p = run.add(made.session(v2), _speech(452))
    cap = engine.session_io_geometry(a)['max_out']
    rid = engine.reblock_create(FS // 4, cap, 80.0)
    made.reblocks.append(rid)
    run.attach(a, rid)
    gid = made.group([p])
    for t in range(10):
        if t == 3:
            run.change(lambda: engine.group_add(gid, a))
        if t == 7:
            run.change(lambda: engine.group_remove(gid, a))
        run.group(gid)
        if t < 3 or t >= 7:
            run.alone(a)
    run.drain()
    host = engine.reblock_create(FS // 4, cap, 80.0)
    made.reblocks.append(host)
    assert len(run.rb[a]) == len(run.outs[a]) == 10
    for k, y in enumerate(run.outs[a]):
        st, chunk, power = engine.reblock_push(host, y)
        got = run.rb[a][k]
        assert got[0] == st and got[2] == power, k
        assert (chunk is None) == (got[1] is None), k
        if chunk is not None:
            assert np.array_equal(got[1], chunk), k
