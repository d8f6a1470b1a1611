"""A CPU stand-in for realtime_yukarin_b200.engine.Engine built on the oracle -- TESTS ONLY.
It lets the host-side Stream/VoiceChanger/Vocoder logic be checked end to end without a GPU
(the product never uses it; the product path raises when libryk / an H100 is missing)."""
import numpy as np

from oracle import nets as onets
from oracle import pipeline as opipe
from oracle import world as W


class OracleEngine:
    def __init__(self, stage1_npz, stage2_npz, cfg=None, backend='torch'):
        self.cfg = cfg or opipe.PathConfig()
        self.p1, self.p2 = onets.load_npz(stage1_npz), onets.load_npz(stage2_npz)
        self.backend = backend
        self.stats = None
        self.synths = {}

    # model upload is a no-op: the oracle reads the same npz files
    def model_create(self, *a):
        pass

    def model_layer_shape(self, stage, layer):
        p = self.p1 if stage == 1 else self.p2
        part, i = ('encoder', layer) if layer < 8 else ('decoder', layer - 8)
        plain = (part == 'encoder' and i == 0) or (part == 'decoder' and i == 7)
        Wt = p[f'{part}/c{i}/W'] if plain else p[f'{part}/c{i}/c/W']
        tr = part == 'decoder' and i < 7
        cin, cout = (Wt.shape[0], Wt.shape[1]) if tr else (Wt.shape[1], Wt.shape[0])
        return tr, cin, cout, Wt.shape[-1]

    def model_set_layer(self, *a):
        pass

    def stage1_set_stats(self, *a):
        pass

    def f0_set_stats(self, *stats):
        self.stats = stats

    def world_analyze(self, x, fs, frame_period, f0_floor, f0_ceil, fft_length, order, alpha, f0=None):
        f = opipe.extract_features(np.asarray(x, np.float32), self.cfg)
        return dict(f0=f['f0'].ravel(), sp=f['sp'], ap=f['ap'], mc=f['mc'], voiced=f['voiced'].ravel())

    def convert_window(self, wave, fs, frame_length, hop, threshold_db, f0, ap, mc, voiced, order, alpha, fftlen):
        feat = dict(f0=np.asarray(f0, np.float32).reshape(-1, 1), ap=ap, mc=mc, voiced=np.asarray(voiced, bool).reshape(-1, 1))
        out = opipe.convert_window(np.asarray(wave, np.float32), feat, self.cfg, self.p1, self.p2, self.stats, self.backend,
                                   threshold_db=threshold_db)
        return dict(f0=out['f0'].ravel(), ap=out['ap'], sp=out['sp'], voiced=out['voiced'].ravel(), mc=out['mc'])

    def silence_mask(self, wave, frame_length, hop, threshold_db, n_frames):
        return opipe.effective_mask(np.asarray(wave, np.float32), n_frames, self.cfg, threshold_db)

    def stage1_convert(self, x):
        return onets.stage1_convert(x, self.p1, self.backend)

    def f0_convert(self, f0, voiced):
        return opipe.f0_convert(f0, voiced, self.stats)

    def mc2sp(self, mc, alpha, fftlen):
        return W.mc2sp(np.asarray(mc, np.float32), alpha, fftlen)

    def stage2_convert(self, sp):
        return onets.stage2_convert(sp, self.p2, self.backend)

    def synth_create(self, fs, frame_period, fft_size, buffer_size, number_of_pointers=16):
        self.synths[len(self.synths)] = W.RealtimeSynthesizer(fs, frame_period, fft_size, buffer_size)
        return len(self.synths) - 1

    def synth_decode(self, sid, f0, sp, ap, max_blocks=None):
        return self.synths[sid].decode(np.asarray(f0, np.float64).ravel(), sp, ap)

    def synth_destroy(self, sid):
        self.synths.pop(sid, None)

    # ---- SURVEY 8(f) ranks 2 / 3: offline synthesis, output gate and re-blocker ----
    def world_synthesize(self, f0, sp, ap, fs, frame_period, fft_size=None, return_pulses=False):
        return W.synthesize(f0, sp, ap, fs, frame_period, fft_size, return_pulses)

    def output_gate(self, wave, threshold_db, n_fft=2048, hop=512):
        pw = W.stft_power_db_mean(wave, n_fft, hop)
        return pw, not (pw < -threshold_db)

    def reblock_create(self, out_audio_chunk, max_in, threshold_db, n_fft=2048, hop=512):
        self.reblocks = getattr(self, 'reblocks', {})
        self.reblocks[len(self.reblocks)] = opipe.OutputReblockOracle(out_audio_chunk, threshold_db)
        return len(self.reblocks) - 1

    def reblock_push(self, rid, wave):
        st, chunk = self.reblocks[rid].push(wave)
        return st, chunk, self.reblocks[rid].last_power or 0.0

    def reblock_destroy(self, rid):
        self.reblocks.pop(rid, None)

    def resample_poly(self, x, up, down, taps):
        import scipy.signal as ss
        return ss.resample_poly(np.asarray(x, np.float64), up, down, window=np.asarray(taps, np.float64) / up).astype(np.float32)

    # ---- device-session stand-in (worker.RealtimePipeline on CPU): StreamOracle + OutputReblockOracle, results kept per ticket ----
    def session_create(self, cfg):
        self.sessions = getattr(self, 'sessions', {})
        sid = len(self.sessions)
        stats = self.stats if self.stats is not None else (float(np.log(150.0)), 0.2, float(np.log(250.0)), 0.2)
        pc = opipe.PathConfig(frame_period=cfg.frame_period_ms, threshold_db=cfg.threshold_db)
        orc = opipe.StreamOracle(pc, self.p1, self.p2, stats, buffer_time=cfg.buffer_time,
                                 extra=(cfg.encode_extra_time, cfg.convert_extra_time, cfg.decode_extra_time), backend=self.backend)
        self.sessions[sid] = dict(orc=orc, out={}, step=0, last=None)
        return sid

    def session_submit(self, sid, wave):
        S = self.sessions[sid]
        S['last'] = S['orc'].push(np.asarray(wave, np.float32))
        S['out'][S['step']] = S['last']
        S['step'] += 1
        return S['step'] - 1

    def session_collect(self, sid, ticket, out):
        y = self.sessions[sid]['out'].pop(ticket)
        out[:len(y)] = y
        return out[:len(y)]

    def session_poll(self, sid, ticket):
        return True                      # the stand-in computes synchronously in submit

    def reblock_poll(self, rid, ticket):
        return True

    def session_destroy(self, sid):
        self.sessions.pop(sid, None)

    def reblock_push_device(self, rid, session_id=-1, wave_dev_ptr=0, n_dev_ptr=0):
        assert session_id >= 0, 'the stand-in only supports the attached mode'
        R = self.reblocks[rid]
        res = getattr(R, 'results', None)
        if res is None:
            res = R.results = {}
            R.pushed = 0
        st, chunk = R.push(self.sessions[session_id]['last'])
        res[R.pushed] = (st, chunk, R.last_power or 0.0)
        R.pushed += 1
        return R.pushed - 1

    def reblock_collect(self, rid, ticket):
        return self.reblocks[rid].results.pop(ticket)
