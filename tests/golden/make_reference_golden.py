"""Regenerates the fixtures that pin this package against the original project (Hiroshiba/realtime-yukarin):

  reference_golden.npz          outputs of the original's own code (check.py, stream / voice-changer glue, workers) over this
                                package's replacements, as the tests in test_stream_api.py / test_reference_glue_differential.py drove
                                it; arrays are stored as digests (shape + a fixed, seeded sample of elements)
  reference_fetch_golden.json   segment layouts / fetch windows / remove times and the original BaseStream's answers (sha256)
  reference_config.yaml         the original's config.yaml (data)
  reference_config_fields.json  what the original's Config.from_yaml reads from it
  audioA_24k_4s.wav             the first 4 s of the original's tests/data/audioA.wav, resampled to 24 kHz (16-bit PCM)

usage: python tests/golden/make_reference_golden.py <checkout of the original project>
The tests only read these files; nothing here runs during the suite."""
import hashlib
import importlib
import json
import queue
import shutil
import sys
import tempfile
import threading
import types
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE.parent.parent))
DIGEST_N = 128


def digest(prefix, a, out):
    """shape + DIGEST_N elements at seeded flat positions (all of them when the array is smaller)"""
    a = np.asarray(a, dtype=np.float64)
    out[prefix + '/shape'] = np.asarray(a.shape, np.int64)
    idx = np.arange(a.size) if a.size <= DIGEST_N else np.sort(np.random.default_rng(a.size).choice(a.size, DIGEST_N, replace=False))
    out[prefix + '/idx'] = idx.astype(np.int64)
    out[prefix + '/val'] = a.ravel()[idx]


def check_digest(g, prefix, a, atol=0.0, rtol=0.0):
    """assert that `a` matches the stored digest (NaN where the original had NaN; elsewhere |diff| <= atol + rtol * the largest
    stored magnitude)"""
    a = np.asarray(a, dtype=np.float64)
    assert tuple(a.shape) == tuple(g[prefix + '/shape']), (prefix, a.shape, g[prefix + '/shape'])
    got, want = a.ravel()[g[prefix + '/idx']], g[prefix + '/val']
    assert np.array_equal(np.isnan(got), np.isnan(want)), prefix
    ok = ~np.isnan(want)
    tol = atol + rtol * (np.abs(want[ok]).max() if ok.any() else 0.0)
    assert np.all(np.abs(got[ok] - want[ok]) <= tol), (prefix, np.abs(got[ok] - want[ok]).max(), tol)


def array_sha(a):
    return hashlib.sha256(np.ascontiguousarray(np.asarray(a, np.float32)).tobytes()).hexdigest()


def fetch_cases(n=300, seed=11):
    """seeded layouts (gaps, overlaps, touching segments), fetch windows and remove times on the 5 ms grid"""
    rng = np.random.default_rng(seed)
    cases = []
    for _ in range(n):
        layout = [(int(rng.integers(0, 401)) * 0.005, int(rng.integers(1, 301))) for _ in range(int(rng.integers(0, 7)))]
        win = (int(rng.integers(-50, 401)) * 0.005, int(rng.integers(1, 201)) * 0.005, int(rng.integers(0, 101)) * 0.005)
        rm = None if rng.random() < 0.5 else int(rng.integers(0, 401)) * 0.005
        cases.append(dict(rate=int(rng.choice([200, 1000, 24000])), layout=sorted(layout), win=win, rm=rm))
    return cases


def run_fetch_case(BaseStream, make_method, c):
    """-> (start times left after remove (or None), fetched array)"""
    s = BaseStream(in_segment_method=make_method(c['rate']), out_segment_method=make_method(c['rate']))
    base = 1.0
    for start, n_frames in c['layout']:
        n = round(n_frames * 0.005 * c['rate'])
        s.add(start_time=start, data=(base + np.arange(n)).astype(np.float32))
        base += 100000.0
    left = None
    if c['rm'] is not None:
        s.remove(end_time=c['rm'])
        left = [seg.start_time for seg in s.stream]
    return left, s.fetch(start_time=c['win'][0], time_length=c['win'][1], extra_time=c['win'][2])


def small_models(d):
    from realtime_yukarin_b200.synthetic import write_synthetic_models
    return write_synthetic_models(d, seed=3, base1=16, base2=16)          # the suite's `small_models` fixture


class RealPackage:
    """`realtime_voice_conversion` resolves to the original's files, except yukarin_wrapper.vocoder (the pyworld / world4py
    binding), which is this package's."""

    def __init__(self, root):
        self.root = Path(root)

    def __enter__(self):
        from realtime_yukarin_b200 import dropin, vocoder
        dropin.install()
        self.saved = {k: v for k, v in sys.modules.items() if k.split('.')[0] in ('realtime_voice_conversion', 'librosa', 'chainer')}
        for k in self.saved:
            del sys.modules[k]
        pkg = types.ModuleType('realtime_voice_conversion')
        pkg.__path__ = [str(self.root / 'realtime_voice_conversion')]
        sys.modules['realtime_voice_conversion'] = pkg
        yw = types.ModuleType('realtime_voice_conversion.yukarin_wrapper')
        yw.__path__ = [str(self.root / 'realtime_voice_conversion' / 'yukarin_wrapper')]
        sys.modules['realtime_voice_conversion.yukarin_wrapper'] = yw
        voc = types.ModuleType('realtime_voice_conversion.yukarin_wrapper.vocoder')
        voc.Vocoder, voc.RealtimeVocoder = vocoder.Vocoder, vocoder.RealtimeVocoder
        sys.modules['realtime_voice_conversion.yukarin_wrapper.vocoder'] = voc
        from tests.test_reference_glue_differential import librosa_module
        lib, core = librosa_module()
        sys.modules['librosa'], sys.modules['librosa.core'] = lib, core
        chainer = types.ModuleType('chainer')
        chainer.global_config = types.SimpleNamespace(enable_backprop=True, train=True)
        sys.modules['chainer'] = chainer
        return self

    def load(self, name):
        return importlib.import_module(f'realtime_voice_conversion.{name}')

    def __exit__(self, *exc):
        for k in [k for k in sys.modules if k.split('.')[0] in ('realtime_voice_conversion', 'librosa', 'chainer')]:
            del sys.modules[k]
        sys.modules.update(self.saved)
        return False


def main(root):
    import scipy.signal
    from realtime_yukarin_b200 import engine as eng_mod
    from realtime_yukarin_b200 import synthetic, wave_io
    from tests import test_reference_glue_differential as glue
    from tests.fake_engine import OracleEngine
    root = Path(root)
    out = {}

    # ---- audio and configuration data ----
    data, fs = wave_io.read_wav(root / 'tests' / 'data' / 'audioA.wav')
    x = data.astype(np.float64)
    if x.ndim > 1:
        x = x.mean(axis=1)
    x = scipy.signal.resample_poly(x, 24000, fs)[:24000 * 4]
    import wave
    with wave.open(str(HERE / 'audioA_24k_4s.wav'), 'wb') as w:          # 16-bit PCM, like the original recording
        w.setnchannels(1); w.setsampwidth(2); w.setframerate(24000)
        w.writeframes(np.clip(np.round(x * 32768.0), -32768, 32767).astype('<i2').tobytes())
    shutil.copyfile(root / 'config.yaml', HERE / 'reference_config.yaml')

    with RealPackage(root) as ref:
        rc = ref.load('config')
        a = rc.Config.from_yaml(HERE / 'reference_config.yaml')
        fields = {n: (getattr(a, n).value if hasattr(getattr(a, n), 'value') else getattr(a, n)) for n in a._fields}
        fields = {k: (str(v) if isinstance(v, Path) else v) for k, v in fields.items()}
        fields['in_audio_chunk'], fields['out_audio_chunk'] = a.in_audio_chunk, a.out_audio_chunk
    (HERE / 'reference_config_fields.json').write_text(json.dumps(fields, indent=1, sort_keys=True) + '\n')

    # ---- BaseStream fetch / remove ----
    seg_path = root / 'realtime_voice_conversion'
    pkg = types.ModuleType('realtime_voice_conversion'); pkg.__path__ = []
    sub = types.ModuleType('realtime_voice_conversion.segment'); sub.__path__ = []
    sys.modules['realtime_voice_conversion'], sys.modules['realtime_voice_conversion.segment'] = pkg, sub
    spec = importlib.util.spec_from_file_location('realtime_voice_conversion.segment.segment', seg_path / 'segment' / 'segment.py')
    seg = importlib.util.module_from_spec(spec); sys.modules['realtime_voice_conversion.segment.segment'] = seg; spec.loader.exec_module(seg)
    spec = importlib.util.spec_from_file_location('_ref_base_stream', seg_path / 'stream' / 'base_stream.py')
    bs = importlib.util.module_from_spec(spec); spec.loader.exec_module(bs)
    for k in ('realtime_voice_conversion', 'realtime_voice_conversion.segment', 'realtime_voice_conversion.segment.segment'):
        sys.modules.pop(k, None)

    class RefWave(seg.BaseSegmentMethod):          # wave_segment.py:8-19 restated on the original's own base class
        def length(self, data): return len(data)
        def pad(self, width): return np.zeros(width, dtype=np.float32)
        def pick(self, data, first, last): return data[first:last]
        def concat(self, datas): return np.concatenate(list(datas))

    cases = fetch_cases()
    for c in cases:
        left, got = run_fetch_case(bs.BaseStream, RefWave, c)
        c['left'], c['len'], c['sha256'] = left, int(len(got)), array_sha(got)
    (HERE / 'reference_fetch_golden.json').write_text(json.dumps(cases) + '\n')

    with tempfile.TemporaryDirectory() as td:
        models = small_models(Path(td) / 'models')
        fake = OracleEngine(models['stage1_model_path'], models['stage2_model_path'])
        eng_mod.set_default_engine(fake)
        try:
            # ---- check.py ----
            from realtime_yukarin_b200 import dropin
            dropin.install()
            spec = importlib.util.spec_from_file_location('_reference_check', root / 'check.py')
            check = importlib.util.module_from_spec(spec)
            spec.loader.exec_module(check)
            N = 3
            xs = synthetic.synthetic_speech(N + 0.4, stream=23)
            wave_io.write_wav(Path(td) / 'in.wav', xs, 24000)
            check.check(input_path=Path(td) / 'in.wav', input_time_length=N, output_path=Path(td) / 'out.wav',
                        **{k: models[k] for k in ('input_statistics_path', 'target_statistics_path', 'stage1_model_path',
                                                  'stage1_config_path', 'stage2_model_path', 'stage2_config_path')})
            y, sr = wave_io.read_wav(Path(td) / 'out.wav')
            assert sr == 24000
            digest('check_py/out', y, out)

            # ---- stream + voice-changer glue ----
            for T, extra in glue.STREAM_CASES:
                with RealPackage(root) as ref:
                    rs, rvc = ref.load('stream'), ref.load('yukarin_wrapper.voice_changer')
                    outs = glue.run_stream_chain(models, fake, T, extra, rs.EncodeStream, rs.ConvertStream, rs.DecodeStream,
                                                 rs.StreamWrapper, rvc.VoiceChanger)
                tag = glue.stream_tag(T, extra)
                out[tag + '/chunks'] = np.asarray(len(outs))
                for i, arrs in enumerate(outs):
                    for j, a in enumerate(arrs):
                        digest(f'{tag}/{i}/{j}', a, out)

            # ---- the three workers ----
            cfg, x_w, K, played_max = glue.worker_setup(models, fake)
            with RealPackage(root) as ref:
                workers = ref.load('worker')
                q_in, q_feat, q_conv, q_out = queue.Queue(), queue.Queue(), queue.Queue(), queue.Queue()
                locks = [threading.Lock() for _ in range(3)]
                for lk in locks:
                    lk.acquire()
                ac, srn, acp, voc = glue.worker_models(models, fake)
                T, extra = glue.WORKER_T, glue.WORKER_EXTRA
                threads = [
                    threading.Thread(target=workers.encode_worker, daemon=True, kwargs=dict(
                        realtime_vocoder=voc, time_length=T, extra_time=extra[0], queue_input=q_in, queue_output=q_feat, acquired_lock=locks[0])),
                    threading.Thread(target=workers.convert_worker, daemon=True, kwargs=dict(
                        acoustic_converter=ac, super_resolution=srn, time_length=T, extra_time=extra[1],
                        input_silent_threshold=cfg.input_silent_threshold, queue_input=q_feat, queue_output=q_conv, acquired_lock=locks[1])),
                    threading.Thread(target=workers.decode_worker, daemon=True, kwargs=dict(
                        realtime_vocoder=voc, time_length=T, extra_time=extra[2], vocoder_buffer_size=1024, out_audio_chunk=cfg.out_audio_chunk,
                        output_silent_threshold=cfg.output_silent_threshold, queue_input=q_conv, queue_output=q_out, acquired_lock=locks[2])),
                ]
                for th in threads:
                    th.start()
                for lk in locks:
                    assert lk.acquire(timeout=30)
                Item = ref.load('worker.utility').Item
                n = round(T * 24000)
                items = []
                for k in range(K):
                    q_in.put(Item(item=x_w[k * n:(k + 1) * n].copy(), index=k))
                    items.append(q_out.get(timeout=120))
            out['workers/index'] = np.asarray([it.index for it in items], np.int64)
            out['workers/played'] = np.asarray([it.item is not None for it in items])
            out['workers/output_silent_threshold'] = np.asarray(cfg.output_silent_threshold)
            for k, it in enumerate(items):
                if it.item is not None:
                    digest(f'workers/{k}', it.item, out)
        finally:
            eng_mod.set_default_engine(None)
    np.savez_compressed(HERE / 'reference_golden.npz', **out)
    print('wrote', sorted(p.name for p in HERE.glob('reference_*')) + ['audioA_24k_4s.wav'])


if __name__ == '__main__':
    if len(sys.argv) != 2:
        sys.exit(__doc__)
    main(sys.argv[1])
