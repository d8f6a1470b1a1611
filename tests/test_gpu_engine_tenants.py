"""One engine serves many callers at once: a session's output must not depend on what else the engine runs.

Every session captures its stage graphs once, at creation, with the device pointers of that moment; the per-op API (world_analyze,
mc2sp, convert_window, ...) runs on the engine's own stream in between.  Engine state that one caller replaces while another's graphs
still point at it shows up here as a difference:

  * tenants: a roster of heterogeneous sessions (headline FP16 base-64, Harvest, CREPE, device rates, a second voice, a mixed-voice
    group, the layered stage 1, a re-blocker attached to a session) is run twice, each tenant alone on the engine and all of them
    together, stepped round-robin with up to 4 chunks in flight each.  Every step's output is bitwise the same in both runs;
  * between the steps of the together run the per-op API is called at other SPTK keys (order, alpha, fft), voices and sessions are
    created and destroyed, and the precision is switched for a moment.  Each call's result is bitwise the result of the same call on
    the quiet engine, and that result matches the FP64 oracle at the tolerance the parity tests use for the call;
  * without sessions, mc2sp and world_analyze alternate across SPTK keys and each matches the oracle at its own key.

The module shares the engine with later modules: it loads voice 0 before any session exists, and destroys everything it makes and
restores the precision (fp16), the f0 method (dio) and the fused stage 1 whatever fails.
"""
import itertools

import numpy as np
import pytest
import scipy.signal as ss

from oracle import crepe as oc
from oracle import nets as onets
from oracle import pipeline as opipe
from oracle import world as oworld
from realtime_yukarin_b200 import crepe as pcrepe
from realtime_yukarin_b200 import synthetic, wave_io

pytestmark = pytest.mark.gpu

FS = 24000
CFG = opipe.PathConfig()
CFG48 = opipe.PathConfig(fs=48000, fft_length=2048)
STEPS = 10
DEPTH = 3                   # chunks submitted ahead of the one collected: up to 4 in flight per tenant
# (order, alpha, fft) keys of the SPTK conversions: every order 8 / 24 / 39, alpha 0.35 / 0.42 / 0.466 / 0.544 and fft 1024 / 2048
SPTK_KEYS = [(8, 0.466, 1024), (24, 0.35, 2048), (39, 0.544, 1024), (8, 0.42, 2048), (24, 0.466, 1024), (39, 0.42, 2048),
             (8, 0.544, 1024), (24, 0.544, 2048), (39, 0.35, 1024), (8, 0.35, 1024), (39, 0.466, 2048), (24, 0.42, 1024)]


def _cfg(T, extra=(0.0, 0.5, 0.0), alpha=0.466):
    from realtime_yukarin_b200.engine import SessionConfig
    return SessionConfig(fs=FS, frame_period_ms=5.0, f0_floor=71.0, f0_ceil=800.0, fft_length=1024, order=8, alpha=alpha,
                         buffer_time=T, encode_extra_time=extra[0], convert_extra_time=extra[1], decode_extra_time=extra[2],
                         threshold_db=60.0, vocoder_buffer_size=1024)


def _same(a, b):
    """Bitwise equality of nested lists / tuples / dicts of arrays and scalars (NaN payloads included)."""
    if isinstance(a, dict):
        return isinstance(b, dict) and a.keys() == b.keys() and all(_same(a[k], b[k]) for k in a)
    if isinstance(a, (list, tuple)):
        return isinstance(b, (list, tuple)) and len(a) == len(b) and all(_same(x, y) for x, y in zip(a, b))
    if a is None or b is None:
        return a is None and b is None
    a, b = np.asarray(a), np.asarray(b)
    return a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()


def _logspec_err(a, b):
    d = np.log(np.asarray(a, np.float64)) - np.log(np.asarray(b, np.float64))
    return float(np.sqrt((d ** 2).mean(axis=1)).max()), float(np.abs(d).max())


def _check_analysis(got, ref):
    """world_analyze against extract_features, at the tolerances of test_gpu_parity.test_world_analysis_matches_oracle."""
    f0r, f0g = ref['f0'].ravel(), got['f0']
    assert np.array_equal(f0r != 0, f0g != 0)
    assert np.allclose(f0g, f0r, rtol=1e-6, atol=0)
    assert np.array_equal(ref['voiced'].ravel(), got['voiced'])
    assert np.allclose(np.log(got['sp']), np.log(ref['sp']), atol=2e-4), np.abs(np.log(got['sp']) - np.log(ref['sp'])).max()
    assert np.allclose(got['ap'], ref['ap'], rtol=1e-4, atol=1e-6), np.abs(got['ap'] - ref['ap']).max()
    assert np.allclose(got['mc'], ref['mc'], atol=2e-4), np.abs(got['mc'] - ref['mc']).max()


def _mc(T, order, seed):
    """Mel-cepstra with the decay of real ones: c0 around -5, c_j of scale 0.5 / (1 + j)."""
    rng = np.random.default_rng(seed)
    mc = rng.standard_normal((T, order + 1)) * (0.5 / (1.0 + np.arange(order + 1)))
    mc[:, 0] += -5.0
    return mc.astype(np.float32)


def _analyze(engine, x, cfg, order=None, alpha=None):
    return engine.world_analyze(x, cfg.fs, cfg.frame_period, cfg.f0_floor, cfg.f0_ceil, cfg.fft_length,
                                cfg.order if order is None else order, cfg.alpha if alpha is None else alpha)


def _load_voice(engine, paths, voice):
    from realtime_yukarin_b200.models import load_voice
    load_voice(engine, voice, **{k: paths[k] for k in ('stage1_model_path', 'stage2_model_path', 'input_statistics_path',
                                                         'target_statistics_path')})


class _Made:
    """Everything the module creates on the shared engine, destroyed in the end whatever fails."""

    def __init__(self, engine):
        self.engine, self.groups, self.sessions, self.reblocks, self.voices, self.synths = engine, [], [], [], [], []

    def session(self, cfg, voice=0):
        self.sessions.append(self.engine.session_create(cfg, voice=voice))
        return self.sessions[-1]

    def drop(self, kind, handle, destroy):
        getattr(self, kind).remove(handle)
        destroy(handle)

    def close(self):
        e = self.engine
        for items, destroy in ((self.groups, e.group_destroy), (self.reblocks, e.reblock_destroy), (self.sessions, e.session_destroy),
                               (self.synths, e.synth_destroy), (self.voices, e.voice_destroy)):
            while items:
                destroy(items.pop())


class _Tenant:
    """One session or group of the roster, fed its own chunks; outs[k] = per-member outputs of step k (+ the re-blocker's result)."""

    def __init__(self, name, create, chunks, reblock=False):
        self.name, self.create, self.chunks, self.reblock = name, create, chunks, reblock

    def open(self, made):
        e = made.engine
        self.sids = self.create(made)
        self.gid = None
        if len(self.sids) > 1:
            self.gid = e.group_create(self.sids)
            made.groups.append(self.gid)
        cap = max(e.session_io_geometry(s)['max_out'] for s in self.sids)
        self.bufs = [np.empty(cap) for _ in self.sids]
        self.rid = None
        if self.reblock:
            self.rid = e.reblock_create(FS // 4, cap, 80.0)
            made.reblocks.append(self.rid)
        self.tickets, self.outs = [], []

    def submit(self, engine):
        k = len(self.outs) + len(self.tickets)
        if self.gid is None:
            t = engine.session_submit(self.sids[0], self.chunks[k][0])
        else:
            t = engine.group_submit(self.gid, self.chunks[k])
        rt = engine.reblock_push_device(self.rid, session_id=self.sids[0]) if self.rid is not None else None
        self.tickets.append((t, rt))

    def collect(self, engine):
        t, rt = self.tickets.pop(0)
        if self.gid is None:
            got = [engine.session_collect(self.sids[0], t, self.bufs[0]).copy()]
        else:
            got = [o.copy() for o in engine.group_collect(self.gid, t, self.bufs)]
        if rt is not None:
            st, chunk, power = engine.reblock_collect(self.rid, rt)
            got.append((st, None if chunk is None else chunk.copy(), power))
        self.outs.append(got)

    def step(self, engine):
        self.submit(engine)
        if len(self.tickets) > DEPTH:
            self.collect(engine)

    def drain(self, engine):
        while self.tickets:
            self.collect(engine)

    def close(self, made):
        e = made.engine
        if self.rid is not None:
            made.drop('reblocks', self.rid, e.reblock_destroy)
        if self.gid is not None:
            made.drop('groups', self.gid, e.group_destroy)
        for sid in self.sids:
            made.drop('sessions', sid, e.session_destroy)


def _speech_chunks(T, stream, members=1):
    n = round(T * FS)
    xs = [synthetic.synthetic_speech((STEPS + 1) * T, stream=stream + i) for i in range(members)]
    return [[np.ascontiguousarray(x[k * n:(k + 1) * n]) for x in xs] for k in range(STEPS)]


def _roster(engine, voice1):
    """The tenants (a)-(h); f0 method and stage-1 mode are switched only around the creation that needs them."""
    def single(T, extra=(0.0, 0.5, 0.0), voice=0):
        return lambda made: [made.session(_cfg(T, extra), voice=voice)]

    def harvest(made):
        engine.set_f0_method('harvest')
        try:
            return [made.session(_cfg(0.1, (0.1, 0.2, 0.0)))]
        finally:
            engine.set_f0_method('dio')

    def crepe(made):
        engine.set_f0_method('crepe')
        try:
            return [made.session(_cfg(0.3))]
        finally:
            engine.set_f0_method('dio')

    def rates(made):
        sid = made.session(_cfg(0.3))
        engine.session_set_input_rate(sid, 48000)
        engine.session_set_output_rate(sid, 44100)
        assert engine.session_io_geometry(sid)['n_in'] == n48
        return [sid]

    def group(made):
        return [made.session(_cfg(0.3)), made.session(_cfg(0.3), voice=voice1)]

    def layered(made):
        engine.set_stage1_fused(False)
        try:
            return [made.session(_cfg(0.3))]
        finally:
            engine.set_stage1_fused(True)

    n48 = round(0.3 * 48000)
    x48 = ss.resample_poly(synthetic.synthetic_speech((STEPS + 1) * 0.3, stream=304).astype(np.float64), 2, 1).astype(np.float32)
    return [
        _Tenant('headline', single(0.3), _speech_chunks(0.3, 300)),
        _Tenant('harvest', harvest, _speech_chunks(0.1, 301)),
        _Tenant('crepe', crepe, _speech_chunks(0.3, 302)),
        _Tenant('device rates', rates, [[np.ascontiguousarray(x48[k * n48:(k + 1) * n48])] for k in range(STEPS)]),
        _Tenant('voice 1', single(0.3, voice=voice1), _speech_chunks(0.3, 305)),
        _Tenant('mixed group', group, _speech_chunks(0.3, 306, members=2)),
        _Tenant('layered stage 1', layered, _speech_chunks(0.3, 308)),
        _Tenant('re-blocker', single(0.3), _speech_chunks(0.3, 309), reblock=True),
    ]


def _interference(engine, made, files):
    """(name, call, oracle check) of the per-op calls and lifecycle events made between the together run's steps.  A call returns
    what is compared bitwise with its quiet result; the check asserts the quiet result against the FP64 oracle."""
    paths = files['voice0']
    x24 = synthetic.synthetic_speech(0.6, stream=320)
    x48 = synthetic.synthetic_speech(0.6, stream=321, fs=48000)
    x_cw = synthetic.synthetic_speech(1.3, stream=322)
    enc_cw = opipe.extract_features(x_cw, CFG)
    feat = opipe.extract_features(synthetic.synthetic_speech(0.5, stream=323), CFG)
    rng = np.random.default_rng(324)
    mc_s1 = (synthetic.MC_MEAN_IN + synthetic.MC_STD_IN * rng.standard_normal((128, 9))).astype(np.float32)
    sp_s2 = np.exp(-9 + 2.5 * rng.standard_normal((100, 513))).astype(np.float32)
    x_rs = (rng.standard_normal(9600) * 0.3).astype(np.float32)
    x_gate = rng.standard_normal(7200) * 0.05
    x16 = ss.resample_poly(synthetic.synthetic_speech(0.5, stream=325).astype(np.float64), 2, 3).astype(np.float32)
    chunks_extra = _speech_chunks(0.3, 326)[:2]
    p1, p2 = onets.load_npz(paths['stage1_model_path']), onets.load_npz(paths['stage2_model_path'])
    from realtime_yukarin_b200.models import F0Converter
    f0c = F0Converter(paths['input_statistics_path'], paths['target_statistics_path'])
    fft = oworld.cheaptrick_fft_size(FS)
    calls = []

    def add(name, call, check):
        calls.append((name, call, check))

    add('world_analyze 24 kHz', lambda: _analyze(engine, x24, CFG), lambda got: _check_analysis(got, opipe.extract_features(x24, CFG)))
    add('world_analyze 48 kHz', lambda: _analyze(engine, x48, CFG48), lambda got: _check_analysis(got, opipe.extract_features(x48, CFG48)))
    for i, (order, alpha, nfft) in enumerate(SPTK_KEYS):
        mc = _mc(40, order, 330 + i)

        def check_mc2sp(got, mc=mc, alpha=alpha, nfft=nfft):
            ref = oworld.mc2sp(mc, alpha, nfft)
            assert np.allclose(np.log(got), np.log(ref), atol=1e-9), np.abs(np.log(got) - np.log(ref)).max()
        add(f'mc2sp {(order, alpha, nfft)}', lambda mc=mc, alpha=alpha, nfft=nfft: engine.mc2sp(mc, alpha, nfft), check_mc2sp)

    def check_s1(got):
        err = float(np.abs(got - onets.stage1_convert(mc_s1, p1, backend='torch')).max())
        assert err < 2e-2, err

    def check_s2(got):
        l2, mx = _logspec_err(got, onets.stage2_convert(sp_s2, p2, backend='torch'))
        assert l2 <= 1e-2 and mx <= 6e-2, (l2, mx)

    def check_cw(got):
        ref = opipe.convert_window(x_cw, enc_cw, CFG, p1, p2, f0c.stats(), backend='torch')
        assert np.array_equal(np.asarray(got['voiced']).ravel(), ref['voiced'].ravel())
        assert np.allclose(got['f0'], ref['f0'].ravel(), rtol=1e-6)
        l2, mx = _logspec_err(got['sp'], ref['sp'])
        assert l2 <= 1e-2 and mx <= 6e-2, (l2, mx)
    add('stage1_convert', lambda: engine.stage1_convert(mc_s1), check_s1)
    add('stage2_convert', lambda: engine.stage2_convert(sp_s2), check_s2)
    add('convert_window', lambda: engine.convert_window(x_cw, CFG.fs, CFG.fft_length, CFG.hop, 60.0, enc_cw['f0'].ravel(), enc_cw['ap'],
                                                        enc_cw['mc'], enc_cw['voiced'].ravel(), CFG.order, CFG.alpha, CFG.fft_length),
        check_cw)

    f0 = feat['f0'].ravel().astype(np.float64)

    def check_synthesize(got):
        ref = oworld.synthesize(f0, feat['sp'], feat['ap'], FS, 5.0)
        assert len(got) == len(ref)
        assert float(np.sqrt(np.mean((got - ref) ** 2))) <= 1e-9 * max(1.0, float(np.abs(ref).max()))

    def synth_cycle():
        sid = engine.synth_create(FS, 5.0, fft, 1024)
        made.synths.append(sid)
        y = engine.synth_decode(sid, f0, feat['sp'], feat['ap'])
        made.drop('synths', sid, engine.synth_destroy)
        return y

    def check_synth(got):
        ref = oworld.RealtimeSynthesizer(FS, 5.0, fft, 1024).decode(f0, feat['sp'], feat['ap'])
        assert len(got) == len(ref) and len(ref) > 0
        assert float(np.sqrt(np.mean((got - ref) ** 2))) < 1e-6 * max(1.0, float(np.abs(ref).max()) * 1e3)
    add('world_synthesize', lambda: engine.world_synthesize(f0, feat['sp'], feat['ap'], FS, 5.0), check_synthesize)
    add('synthesizer create / decode / destroy', synth_cycle, check_synth)

    taps = wave_io.resample_filter(1, 2)

    def check_resample(got):
        ref = ss.resample_poly(x_rs.astype(np.float64), 1, 2, window=taps)       # up = 1: the taps are the window
        assert len(got) == len(ref)
        assert np.abs(got - ref).max() < 1e-6 * max(1.0, float(np.abs(ref).max()))

    def check_gate(got):
        ref = oworld.stft_power_db_mean(x_gate)
        assert abs(got[0] - ref) < 1e-9 and got[1] == (not ref < -80.0), (got, ref)
    add('resample_poly 48 -> 24 kHz', lambda: engine.resample_poly(x_rs, 1, 2, taps), check_resample)
    add('output_gate', lambda: engine.output_gate(x_gate, 80.0), check_gate)

    w_crepe = dict(np.load(files['crepe']))

    def check_crepe(got):
        act = got[3]
        err = float(np.abs(act - oc.get_activation(x16, w_crepe, 5.0)).max())
        assert err < 5e-4, err
    add('crepe.predict', lambda: pcrepe.predict(x16, 16000, step_size=5.0, engine=engine, details=True), check_crepe)

    def voice_cycle():
        v = engine.voice_create()
        made.voices.append(v)
        _load_voice(engine, files['narrow'], v)
        made.drop('voices', v, engine.voice_destroy)

    def extra_session(precision, alpha):
        def run():
            engine.set_precision(precision)
            try:
                sid = made.session(_cfg(0.3, alpha=alpha))
                out = [engine.session_push(sid, c[0]).copy() for c in chunks_extra]
                made.drop('sessions', sid, engine.session_destroy)
                return out
            finally:
                engine.set_precision('fp16')
        return run

    def check_extra(got):
        assert sum(len(o) for o in got) > 0
    add('voice create / load / destroy', voice_cycle, lambda got: None)
    add('session at alpha 0.42', extra_session('fp16', 0.42), check_extra)
    add('fp32 session', extra_session('fp32', 0.466), check_extra)
    return calls


@pytest.fixture(scope='module')
def files(tmp_path_factory):
    """Voice 0 and voice 1 (base 64, seeds 20 and 21), a base-16 voice for the create / destroy cycles, tiny CREPE weights."""
    d = tmp_path_factory.mktemp('tenants')
    return {'voice0': synthetic.write_synthetic_models(d / 'v0', seed=20), 'voice1': synthetic.write_synthetic_models(d / 'v1', seed=21),
            'narrow': synthetic.write_synthetic_models(d / 'narrow', seed=22, base1=16, base2=16),
            'crepe': synthetic.write_crepe_model(d / 'crepe', seed=5, capacity='tiny')}


def test_tenants_are_bitwise_their_runs_alone(engine, files):
    import time
    t_start = time.perf_counter()
    made = _Made(engine)
    try:
        engine.set_precision('fp16')
        engine.set_f0_method('dio')
        engine.set_stage1_fused(True)
        _load_voice(engine, files['voice0'], 0)
        pcrepe.load_crepe_model(files['crepe'], engine)
        voice1 = engine.voice_create()
        made.voices.append(voice1)
        _load_voice(engine, files['voice1'], voice1)
        calls = _interference(engine, made, files)

        # the per-op calls on the quiet engine, each checked against the oracle
        quiet = {}
        for name, call, check in calls:
            quiet[name] = call()
            check(quiet[name])

        # each tenant alone
        tenants = _roster(engine, voice1)
        alone = {}
        for t in tenants:
            t.open(made)
            for _ in range(STEPS):
                t.step(engine)
            t.drain(engine)
            t.close(made)
            alone[t.name] = t.outs
            assert sum(len(o) for step in t.outs for o in step[:len(t.sids)]) > 0, t.name

        # all together, with a per-op call or lifecycle event after every step of every tenant
        ops = itertools.cycle(calls)
        made_calls = {}
        for t in tenants:
            t.open(made)
        for _ in range(STEPS):
            for t in tenants:
                t.step(engine)
                name, call, _ = next(ops)
                got = call()
                assert _same(got, quiet[name]), f'{name}: differs from the same call on the quiet engine'
                made_calls[name] = made_calls.get(name, 0) + 1
        for t in tenants:
            t.drain(engine)
        for t in tenants:
            t.close(made)
        assert set(made_calls) == set(quiet)
        for t in tenants:
            assert len(t.outs) == STEPS
            for k in range(STEPS):
                assert _same(t.outs[k], alone[t.name][k]), f'{t.name}: step {k} differs from its run alone'
        print(f'{len(tenants)} tenants x {STEPS} steps, {sum(made_calls.values())} calls / events in between: bitwise their runs alone '
              f'({time.perf_counter() - t_start:.1f} s)')
    finally:
        made.close()
        engine.set_precision('fp16')
        engine.set_f0_method('dio')
        engine.set_stage1_fused(True)


def test_sptk_keys_alternate_without_sessions(engine):
    """mc2sp and world_analyze alternate across (order, alpha, fft) keys: each call converts with its own key's matrices."""
    x24 = synthetic.synthetic_speech(0.4, stream=340)
    x48 = synthetic.synthetic_speech(0.4, stream=341, fs=48000)
    for rnd in range(2):
        for i, (order, alpha, nfft) in enumerate(SPTK_KEYS):
            mc = _mc(30, order, 350 + i)
            got = engine.mc2sp(mc, alpha, nfft)
            ref = oworld.mc2sp(mc, alpha, nfft)
            assert np.allclose(np.log(got), np.log(ref), atol=1e-9), ((order, alpha, nfft), np.abs(np.log(got) - np.log(ref)).max())
            # world_analyze at the key the previous mc2sp did not use
            order2, alpha2, nfft2 = SPTK_KEYS[(i + 1 + rnd) % len(SPTK_KEYS)]
            cfg = opipe.PathConfig(fs=24000 if nfft2 == 1024 else 48000, fft_length=nfft2, order=order2, alpha=alpha2)
            x = x24 if nfft2 == 1024 else x48
            got = _analyze(engine, x, cfg)
            assert got['mc'].shape[1] == order2 + 1
            _check_analysis(got, opipe.extract_features(x, cfg))
