"""ctypes binding of libryk.so (include/ryk.h): the only door between the Python host layer and
the CUDA hot path.  There is NO CPU fallback: if the shared object is missing, cannot be loaded, or
no H100 is visible, every call raises.
"""
import os as _os

# must be in the environment before the CUDA context exists (see ryk_engine_create): many independent streams need their own hardware queues
_os.environ.setdefault('CUDA_DEVICE_MAX_CONNECTIONS', '32')

import ctypes
import math
import os
import threading
from pathlib import Path
from typing import Dict, List, Optional, Sequence

import numpy

from .world_consts import cheaptrick_fft_size, dio_num_frames  # noqa: F401  (re-exported)

_CSRC = Path(__file__).resolve().parent / 'csrc'
_LIB_PATH = Path(os.environ['RYK_LIB']) if os.environ.get('RYK_LIB') else _CSRC / 'libryk.so'     # RYK_LIB: diagnostics builds

c_int_p = ctypes.POINTER(ctypes.c_int)
c_float_p = ctypes.POINTER(ctypes.c_float)
c_double_p = ctypes.POINTER(ctypes.c_double)
c_u8_p = ctypes.POINTER(ctypes.c_uint8)


class RykError(RuntimeError):
    pass


class SessionConfig(ctypes.Structure):
    _fields_ = [
        ('fs', ctypes.c_int), ('frame_period_ms', ctypes.c_double), ('f0_floor', ctypes.c_double),
        ('f0_ceil', ctypes.c_double), ('fft_length', ctypes.c_int), ('order', ctypes.c_int),
        ('alpha', ctypes.c_double), ('buffer_time', ctypes.c_double), ('encode_extra_time', ctypes.c_double),
        ('convert_extra_time', ctypes.c_double), ('decode_extra_time', ctypes.c_double),
        ('threshold_db', ctypes.c_double), ('vocoder_buffer_size', ctypes.c_int),
    ]


_lib = None
_lib_lock = threading.Lock()

# every symbol include/ryk.h declares (tests check that the library exports all of them)
EXPORTED_SYMBOLS = [
    'ryk_abi_version', 'ryk_last_error', 'ryk_engine_create', 'ryk_engine_destroy', 'ryk_engine_set_precision',
    'ryk_engine_get_precision', 'ryk_engine_launch_count', 'ryk_engine_synchronize', 'ryk_world_analyze', 'ryk_world_f0',
    'ryk_world_num_frames', 'ryk_silence_mask', 'ryk_model_create', 'ryk_model_set_layer', 'ryk_model_layer_shape',
    'ryk_stage1_set_stats', 'ryk_f0_set_stats', 'ryk_stage1_convert', 'ryk_f0_convert', 'ryk_mc2sp',
    'ryk_stage2_convert', 'ryk_convert_window', 'ryk_synth_create', 'ryk_synth_destroy', 'ryk_synth_add_parameters',
    'ryk_synth_synthesis2', 'ryk_synth_decode', 'ryk_session_create', 'ryk_session_destroy', 'ryk_session_push',
    'ryk_session_push_device', 'ryk_session_submit', 'ryk_session_collect', 'ryk_group_create', 'ryk_group_destroy',
    'ryk_group_size', 'ryk_session_stage_times', 'ryk_group_submit', 'ryk_group_collect', 'ryk_group_push_device', 'ryk_test_conv_layer', 'ryk_engine_profile', 'ryk_engine_timer_start', 'ryk_engine_timer_stop',
    'ryk_world_synthesize_length', 'ryk_world_synthesize', 'ryk_output_gate', 'ryk_reblock_create', 'ryk_reblock_destroy',
    'ryk_reblock_push', 'ryk_reblock_push_device', 'ryk_reblock_collect', 'ryk_reblock_result_device', 'ryk_resample_length',
    'ryk_resample_poly', 'ryk_session_poll', 'ryk_reblock_poll', 'ryk_engine_profile_read2', 'ryk_engine_set_stage1_fused',
    'ryk_engine_set_f0_method', 'ryk_engine_get_f0_method', 'ryk_debug_harvest',
    'ryk_crepe_create', 'ryk_crepe_set_conv', 'ryk_crepe_set_dense', 'ryk_crepe_set_decoder_tables', 'ryk_crepe_num_frames', 'ryk_crepe_predict',
    'ryk_crepe_set_resampler', 'ryk_crepe_test_conv', 'ryk_crepe_test_network', 'ryk_stage2_row_bands', 'ryk_test_stage2_forward',
    'ryk_stage2_tail_rows',
    'ryk_session_set_input_rate', 'ryk_session_set_output_rate', 'ryk_session_io_geometry',
    'ryk_voice_create', 'ryk_voice_destroy', 'ryk_voice_model_create', 'ryk_voice_model_set_layer', 'ryk_voice_stage1_set_stats',
    'ryk_voice_f0_set_stats', 'ryk_session_create_voice', 'ryk_session_voice', 'ryk_group_add', 'ryk_group_remove', 'ryk_group_members',
    'ryk_session_get_f0_map', 'ryk_session_set_f0_map', 'ryk_session_f0_measure', 'ryk_session_f0_follow', 'ryk_session_f0_measure_reset',
    'ryk_session_f0_measured',
]

SEMITONE = math.log(2.0) / 12.0          # one semitone in ln f0
F0_SD_FLOOR = 0.05                       # follow mode: least in_std (ln f0), about 0.9 semitones


class F0Map(ctypes.Structure):
    """ryk_f0_map: exp((ln f0 - in_mean) / in_std * target_std + target_mean)"""
    _fields_ = [('in_mean', ctypes.c_double), ('in_std', ctypes.c_double), ('target_mean', ctypes.c_double), ('target_std', ctypes.c_double)]
    KEYS = ('in_mean', 'in_std', 'target_mean', 'target_std')


def updated_f0_map(current: Dict[str, float], in_mean=None, in_std=None, target_mean=None, target_std=None,
                   semitones: float = 0.0) -> Dict[str, float]:
    """`current` with the given values replaced (None keeps one) and the target mean raised by `semitones`."""
    new = dict(current)
    for key, value in zip(F0Map.KEYS, (in_mean, in_std, target_mean, target_std)):
        if value is not None:
            new[key] = float(value)
    new['target_mean'] += float(semitones) * SEMITONE
    return new


def stage2_row_bands(Tp: int, W: int, keep_begin: int, keep_len: int) -> numpy.ndarray:
    """[16][2] class-local output rows [y0, y1) that each stage-2 layer computes when rows [keep_begin, keep_begin + keep_len) are
    kept (host only, no device needed)."""
    lib = load_library()
    out = numpy.zeros((16, 2), numpy.int32)
    if lib.ryk_stage2_row_bands(int(Tp), int(W), int(keep_begin), int(keep_len), out.ctypes.data_as(c_int_p)) < 0:
        raise RykError(lib.ryk_last_error().decode('utf-8', 'replace'))
    return out


def stage2_tail_rows(Tp: int, W: int, Tw: int, keep_begin: int, keep_len: int) -> numpy.ndarray:
    """[16][4] (skip_y0, skip_y1, run_y0, run_y1) per stage-2 layer for a window of Tw frames padded to Tp rows with one repeated row:
    the output rows the layer does not compute and the input rows whose load boxes it reads from run_y0 (host only)."""
    lib = load_library()
    out = numpy.zeros((16, 4), numpy.int32)
    if lib.ryk_stage2_tail_rows(int(Tp), int(W), int(Tw), int(keep_begin), int(keep_len), out.ctypes.data_as(c_int_p)) < 0:
        raise RykError(lib.ryk_last_error().decode('utf-8', 'replace'))
    return out


def _unet_layer_shapes(stage: int, in_ch: int, out_ch: int, base: int):
    """(transposed, cin, cout, k) of the 16 layers of a U-Net (csrc/unet.cu unet_create): the layer shapes of a voice >= 1, which the
    C ABI does not report."""
    lvl = [base * m for m in (1, 2, 4, 8, 8, 8, 8, 8)]
    dec = [base * m for m in (8, 8, 8, 8, 4, 2, 1)]
    shapes = [(False, in_ch, base, 3)] + [(False, lvl[i - 1], lvl[i], 4) for i in range(1, 8)]
    shapes += [(True, lvl[7] if d == 0 else dec[d - 1] + lvl[7 - d], dec[d], 4) for d in range(7)]
    return shapes + [(False, 2 * base, out_ch, 3)]


def load_library() -> ctypes.CDLL:
    """dlopen csrc/libryk.so (built by __graft_entry__.build() / csrc/build.sh)."""
    global _lib
    with _lib_lock:
        if _lib is None:
            if not _LIB_PATH.exists():
                raise RykError(f'{_LIB_PATH} is missing: run `python -c "import __graft_entry__ as g; g.build()"` '
                               f'(the hot path has no CPU fallback)')
            # RYK_LIB: another build of the same library (e.g. one compiled with extra nvcc flags); never a different implementation
            lib = ctypes.CDLL(os.environ.get('RYK_LIB') or str(_LIB_PATH))
            lib.ryk_last_error.restype = ctypes.c_char_p
            lib.ryk_engine_launch_count.restype = ctypes.c_longlong
            _lib = lib
    return _lib


def _f32(a) -> numpy.ndarray:
    return numpy.ascontiguousarray(a, dtype=numpy.float32)


def _fp(a: numpy.ndarray):
    return a.ctypes.data_as(c_float_p)


def _dp(a: numpy.ndarray):
    return a.ctypes.data_as(c_double_p)


def _bp(a: numpy.ndarray):
    return a.ctypes.data_as(c_u8_p)


class Engine(object):
    """One per process per GPU (not thread-safe, like the reference's single-threaded stages)."""

    def __init__(self, device: Optional[int] = None):
        self.lib = load_library()
        if device is None:
            device = int(os.environ.get('LOCAL_RANK', '0'))
        self.device = device
        h = ctypes.c_void_p()
        self._check(self.lib.ryk_engine_create(ctypes.c_int(device), ctypes.byref(h)))
        self._h = h
        self._synth_block = {}
        self._reblock_chunk = {}           # re-blocker id -> out_audio_chunk
        self._session_fs = {}              # session id -> the session's (model) rate
        self._voice_shapes = {}            # voice id >= 1 -> stage -> the 16 (transposed, cin, cout, k) of its U-Net

    # ---- plumbing ----
    def _check(self, rc: int):
        if rc < 0:
            raise RykError(self.lib.ryk_last_error().decode('utf-8', 'replace'))
        return rc

    def close(self):
        if getattr(self, '_h', None):
            self.lib.ryk_engine_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_precision(self, mode: str):
        self._check(self.lib.ryk_engine_set_precision(self._h, {'fp32': 0, 'fp16': 1}[mode]))

    def set_stage1_fused(self, enable: bool) -> int:
        """Stage 1 as one cluster kernel (default) or as 16 layer launches; returns the cluster size (<= 0: unavailable)."""
        return int(self.lib.ryk_engine_set_stage1_fused(self._h, 1 if enable else 0))

    @property
    def precision(self) -> str:
        return ['fp32', 'fp16'][self.lib.ryk_engine_get_precision(self._h)]

    @property
    def launch_count(self) -> int:
        """Kernels run by session and group steps so far (synchronises the device)."""
        return self._check(int(self.lib.ryk_engine_launch_count(self._h)))

    def timer_start(self):
        self._check(self.lib.ryk_engine_timer_start(self._h))

    def timer_stop(self) -> float:
        ms = ctypes.c_float()
        self._check(self.lib.ryk_engine_timer_stop(self._h, ctypes.byref(ms)))
        return ms.value

    def profile(self, enable: bool):
        self._check(self.lib.ryk_engine_profile(self._h, int(bool(enable))))

    def profile_read2(self):
        """(sum of per-forward durations ms, union of the intervals ms, forwards) of the stage-2 k4 block since the last read."""
        tot, uni, runs = ctypes.c_double(), ctypes.c_double(), ctypes.c_int()
        self._check(self.lib.ryk_engine_profile_read2(self._h, ctypes.byref(tot), ctypes.byref(uni), ctypes.byref(runs)))
        return tot.value, uni.value, runs.value

    def synchronize(self):
        self._check(self.lib.ryk_engine_synchronize(self._h))

    # ---- WORLD analysis ----
    def world_f0(self, x, fs, frame_period, f0_floor, f0_ceil):
        x = _f32(x)
        n = dio_num_frames(fs, len(x), frame_period)
        f0 = numpy.empty(n, dtype=numpy.float64)
        t = numpy.empty(n, dtype=numpy.float64)
        self._check(self.lib.ryk_world_f0(self._h, _fp(x), len(x), int(fs), ctypes.c_double(frame_period),
                                          ctypes.c_double(f0_floor), ctypes.c_double(f0_ceil), _dp(f0), _dp(t)))
        return f0, t

    def world_analyze(self, x, fs, frame_period, f0_floor, f0_ceil, fft_length, order, alpha, f0=None) -> Dict[str, numpy.ndarray]:
        x = _f32(x)
        hop = int(fs * frame_period / 1000)
        T = len(x) // hop
        nb = fft_length // 2 + 1
        out = dict(
            f0=numpy.zeros(T, dtype=numpy.float32), sp=numpy.zeros((T, nb), dtype=numpy.float32),
            ap=numpy.zeros((T, nb), dtype=numpy.float32), mc=numpy.zeros((T, order + 1), dtype=numpy.float32),
            voiced=numpy.zeros(T, dtype=numpy.uint8))
        f0_arg = None
        if f0 is not None:
            nw = dio_num_frames(fs, len(x), frame_period)
            f0_full = numpy.zeros(nw, dtype=numpy.float64)
            f0_full[:min(nw, len(f0))] = numpy.asarray(f0, dtype=numpy.float64).ravel()[:nw]
            f0_arg = _dp(f0_full)
        if T > 0:
            self._check(self.lib.ryk_world_analyze(
                self._h, _fp(x), len(x), int(fs), ctypes.c_double(frame_period), ctypes.c_double(f0_floor),
                ctypes.c_double(f0_ceil), int(fft_length), int(order), ctypes.c_double(alpha), f0_arg,
                _fp(out['f0']), _fp(out['sp']), _fp(out['ap']), _fp(out['mc']), _bp(out['voiced'])))
        out['voiced'] = out['voiced'].astype(bool)
        return out

    # ---- silence gate ----
    def silence_mask(self, wave, frame_length, hop, threshold_db, n_frames) -> numpy.ndarray:
        w = _f32(wave)
        mask = numpy.zeros(n_frames, dtype=numpy.uint8)
        thr = -1.0 if threshold_db is None else float(threshold_db)
        self._check(self.lib.ryk_silence_mask(self._h, _fp(w), len(w), int(frame_length), int(hop), ctypes.c_double(thr),
                                              int(n_frames), _bp(mask)))
        return mask.astype(bool)

    # ---- voices: voice 0 is the engine's built-in voice (the per-op calls use it); voice_create adds more ----
    def voice_create(self) -> int:
        vid = ctypes.c_int()
        self._check(self.lib.ryk_voice_create(self._h, ctypes.byref(vid)))
        self._voice_shapes[vid.value] = {}
        return vid.value

    def voice_destroy(self, voice: int):
        """Free a voice >= 1 and its weights (fails while a session or group uses it)."""
        self._check(self.lib.ryk_voice_destroy(self._h, int(voice)))
        self._voice_shapes.pop(int(voice), None)

    def session_voice(self, sid: int) -> int:
        return self._check(self.lib.ryk_session_voice(self._h, sid))

    # ---- models (voice 0 goes through the original entry points) ----
    def model_create(self, stage: int, in_channels: int, out_channels: int, base_channels: int, voice: int = 0):
        if voice == 0:
            self._check(self.lib.ryk_model_create(self._h, stage, in_channels, out_channels, base_channels))
            return
        self._check(self.lib.ryk_voice_model_create(self._h, int(voice), stage, in_channels, out_channels, base_channels))
        self._voice_shapes[int(voice)][int(stage)] = _unet_layer_shapes(stage, in_channels, out_channels, base_channels)

    def model_layer_shape(self, stage: int, layer: int, voice: int = 0):
        if voice != 0:
            shapes = self._voice_shapes.get(int(voice), {}).get(int(stage))
            if shapes is None or not 0 <= layer < 16:
                raise RykError(f'voice {voice}: no stage-{stage} model created, or no such layer')
            return shapes[layer]
        tr, cin, cout, k = ctypes.c_int(), ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
        self._check(self.lib.ryk_model_layer_shape(self._h, stage, layer, ctypes.byref(tr), ctypes.byref(cin),
                                                   ctypes.byref(cout), ctypes.byref(k)))
        return bool(tr.value), cin.value, cout.value, k.value

    def model_set_layer(self, stage: int, layer: int, W, scale, shift, voice: int = 0):
        W, scale, shift = _f32(W), _f32(scale), _f32(shift)
        if voice == 0:
            self._check(self.lib.ryk_model_set_layer(self._h, stage, layer, _fp(W), _fp(scale), _fp(shift)))
        else:
            self._check(self.lib.ryk_voice_model_set_layer(self._h, int(voice), stage, layer, _fp(W), _fp(scale), _fp(shift)))

    def stage1_set_stats(self, in_mean, in_std, out_mean, out_std, voice: int = 0):
        a, b, c, d = _f32(in_mean), _f32(in_std), _f32(out_mean), _f32(out_std)
        if voice == 0:
            self._check(self.lib.ryk_stage1_set_stats(self._h, len(a), _fp(a), _fp(b), _fp(c), _fp(d)))
        else:
            self._check(self.lib.ryk_voice_stage1_set_stats(self._h, int(voice), len(a), _fp(a), _fp(b), _fp(c), _fp(d)))

    def f0_set_stats(self, in_mean, in_std, target_mean, target_std, voice: int = 0):
        args = [ctypes.c_double(in_mean), ctypes.c_double(in_std), ctypes.c_double(target_mean), ctypes.c_double(target_std)]
        if voice == 0:
            self._check(self.lib.ryk_f0_set_stats(self._h, *args))
        else:
            self._check(self.lib.ryk_voice_f0_set_stats(self._h, int(voice), *args))

    def stage1_convert(self, x) -> numpy.ndarray:
        x = _f32(x)
        y = numpy.empty_like(x)
        self._check(self.lib.ryk_stage1_convert(self._h, _fp(x), x.shape[0], _fp(y)))
        return y

    def f0_convert(self, f0, voiced) -> numpy.ndarray:
        f = _f32(numpy.asarray(f0).ravel())
        v = numpy.ascontiguousarray(numpy.asarray(voiced).ravel(), dtype=numpy.uint8)
        out = numpy.empty_like(f)
        self._check(self.lib.ryk_f0_convert(self._h, _fp(f), _bp(v), len(f), _fp(out)))
        return out

    def mc2sp(self, mc, alpha, fftlen) -> numpy.ndarray:
        mc = _f32(mc)
        sp = numpy.empty((mc.shape[0], fftlen // 2 + 1), dtype=numpy.float64)
        if mc.shape[0]:
            self._check(self.lib.ryk_mc2sp(self._h, _fp(mc), mc.shape[0], mc.shape[1] - 1, ctypes.c_double(alpha), int(fftlen), _dp(sp)))
        return sp

    def stage2_convert(self, sp) -> numpy.ndarray:
        sp = _f32(sp)
        out = numpy.empty_like(sp)
        self._check(self.lib.ryk_stage2_convert(self._h, _fp(sp), sp.shape[0], _fp(out)))
        return out

    def convert_window(self, wave, fs, frame_length, hop, threshold_db, f0, ap, mc, voiced, order, alpha, fftlen):
        wave, f0, ap, mc = _f32(wave), _f32(numpy.asarray(f0).ravel()), _f32(ap), _f32(mc)
        v = numpy.ascontiguousarray(numpy.asarray(voiced).ravel(), dtype=numpy.uint8)
        T, nb = len(f0), fftlen // 2 + 1
        out = dict(f0=numpy.empty(T, numpy.float32), ap=numpy.empty((T, nb), numpy.float32), sp=numpy.empty((T, nb), numpy.float32),
                   voiced=numpy.empty(T, numpy.uint8), mc=numpy.empty((T, order + 1), numpy.float32))
        thr = -1.0 if threshold_db is None else float(threshold_db)
        self._check(self.lib.ryk_convert_window(
            self._h, _fp(wave), len(wave), int(fs), int(frame_length), int(hop), ctypes.c_double(thr),
            _fp(f0), _fp(ap), _fp(mc), _bp(v), T, int(order), ctypes.c_double(alpha), int(fftlen),
            _fp(out['f0']), _fp(out['ap']), _fp(out['sp']), _bp(out['voiced']), _fp(out['mc'])))
        out['voiced'] = out['voiced'].astype(bool)
        return out

    # ---- synthesizer ----
    def synth_create(self, fs, frame_period, fft_size, buffer_size, number_of_pointers=16) -> int:
        sid = ctypes.c_int()
        self._check(self.lib.ryk_synth_create(self._h, int(fs), ctypes.c_double(frame_period), int(fft_size), int(buffer_size),
                                              int(number_of_pointers), ctypes.byref(sid)))
        self._synth_block[sid.value] = (int(buffer_size), int(fft_size), float(fs) * float(frame_period) / 1000.0)
        return sid.value

    def synth_destroy(self, sid: int):
        self._check(self.lib.ryk_synth_destroy(self._h, sid))

    def synth_add_parameters(self, sid, f0, sp, ap) -> int:
        f0 = numpy.ascontiguousarray(numpy.asarray(f0).ravel(), dtype=numpy.float64)
        sp, ap = _f32(sp), _f32(ap)
        return self._check(self.lib.ryk_synth_add_parameters(self._h, sid, _dp(f0), len(f0), _fp(sp), _fp(ap)))

    def synth_synthesis2(self, sid):
        B = self._synth_block[sid][0]
        buf = numpy.empty(B, dtype=numpy.float64)
        ok = self._check(self.lib.ryk_synth_synthesis2(self._h, sid, _dp(buf)))
        return buf if ok else None

    def synth_decode(self, sid, f0, sp, ap, max_blocks=None) -> numpy.ndarray:
        f0 = numpy.ascontiguousarray(numpy.asarray(f0).ravel(), dtype=numpy.float64)
        sp, ap = _f32(sp), _f32(ap)
        B = self._synth_block[sid][0]
        if max_blocks is None:
            # samples one call can add = frames * (fs * frame_period / 1000) of THIS synthesizer (not a fixed 240 per frame): the
            # reference loops `while _Synthesis2() != 0` until the synthesizer is empty (vocoder.py:103-116)
            max_blocks = max(4, int(len(f0) * self._synth_block[sid][2]) // B + 4)
        out = numpy.empty(max_blocks * B, dtype=numpy.float64)
        nblk = ctypes.c_int()
        self._check(self.lib.ryk_synth_decode(self._h, sid, _dp(f0), len(f0), _fp(sp), _fp(ap), _dp(out), int(max_blocks), ctypes.byref(nblk)))
        return out[:nblk.value * B].copy()

    # ---- offline synthesis (pyworld.synthesize) and the output silence gate / re-blocker ----
    def world_synthesize(self, f0, sp, ap, fs, frame_period, fft_size=None, return_pulses=False):
        """Vocoder.decode's pyworld.synthesize (vocoder.py:50-62): (T,) f0, (T, nb) sp / ap -> float64 wave."""
        f0 = numpy.ascontiguousarray(numpy.asarray(f0).ravel(), dtype=numpy.float64)
        sp, ap = _f32(sp), _f32(ap)
        if fft_size is None:
            fft_size = (sp.shape[1] - 1) * 2
        n = self.lib.ryk_world_synthesize_length(len(f0), ctypes.c_double(frame_period), int(fs))
        y = numpy.zeros(max(n, 1), dtype=numpy.float64)
        cap = max(n, 1) if return_pulses else 1
        idx = numpy.zeros(cap, numpy.int64); shift = numpy.zeros(cap); vuv = numpy.zeros(cap, numpy.int32)
        ny, npulse = ctypes.c_int(), ctypes.c_int()
        self._check(self.lib.ryk_world_synthesize(
            self._h, _dp(f0), len(f0), _fp(sp), _fp(ap), int(fs), ctypes.c_double(frame_period), int(fft_size), _dp(y), len(y), ctypes.byref(ny),
            idx.ctypes.data_as(ctypes.POINTER(ctypes.c_longlong)), _dp(shift), vuv.ctypes.data_as(c_int_p), cap if return_pulses else 0,
            ctypes.byref(npulse)))
        y = y[:ny.value]
        if return_pulses:
            k = min(npulse.value, cap)
            return y, idx[:k], shift[:k], vuv[:k]
        return y

    def output_gate(self, wave, threshold_db, n_fft=2048, hop=512):
        """(mean STFT power in dB, keep?) of one output chunk (decode_worker.py:56-58)."""
        w = numpy.ascontiguousarray(numpy.asarray(wave).ravel(), dtype=numpy.float64)
        pw, ok = ctypes.c_double(), ctypes.c_int()
        self._check(self.lib.ryk_output_gate(self._h, _dp(w), len(w), int(n_fft), int(hop), ctypes.c_double(threshold_db), ctypes.byref(pw),
                                             ctypes.byref(ok)))
        return pw.value, bool(ok.value)

    def reblock_create(self, out_audio_chunk, max_in, threshold_db, n_fft=2048, hop=512) -> int:
        rid = ctypes.c_int()
        self._check(self.lib.ryk_reblock_create(self._h, int(out_audio_chunk), int(max_in), int(n_fft), int(hop), ctypes.c_double(threshold_db),
                                                ctypes.byref(rid)))
        self._reblock_chunk[rid.value] = int(out_audio_chunk)
        return rid.value

    def reblock_destroy(self, rid: int):
        self._check(self.lib.ryk_reblock_destroy(self._h, rid))

    def reblock_push(self, rid: int, wave):
        """Host samples in; returns (status, chunk or None, power_db): status 0 none, 1 chunk, 2 silent chunk (dropped)."""
        w = numpy.ascontiguousarray(numpy.asarray(wave).ravel(), dtype=numpy.float64)
        out = numpy.empty(self._reblock_chunk[rid], dtype=numpy.float64)
        st, pw = ctypes.c_int(), ctypes.c_double()
        self._check(self.lib.ryk_reblock_push(self._h, rid, _dp(w), len(w), _dp(out), ctypes.byref(st), ctypes.byref(pw)))
        return st.value, (out if st.value == 1 else None), pw.value

    def reblock_push_device(self, rid: int, session_id: int = -1, wave_dev_ptr: int = 0, n_dev_ptr: int = 0) -> int:
        ticket = ctypes.c_longlong()
        self._check(self.lib.ryk_reblock_push_device(self._h, rid, int(session_id), ctypes.c_void_p(wave_dev_ptr or None),
                                                     ctypes.c_void_p(n_dev_ptr or None), ctypes.byref(ticket)))
        return ticket.value

    def reblock_collect(self, rid: int, ticket: int):
        out = numpy.empty(self._reblock_chunk[rid], dtype=numpy.float64)
        st, pw = ctypes.c_int(), ctypes.c_double()
        self._check(self.lib.ryk_reblock_collect(self._h, rid, ctypes.c_longlong(ticket), _dp(out), ctypes.byref(st), ctypes.byref(pw)))
        return st.value, (out if st.value == 1 else None), pw.value

    def reblock_poll(self, rid: int, ticket: int) -> bool:
        done = ctypes.c_int()
        self._check(self.lib.ryk_reblock_poll(self._h, rid, ctypes.c_longlong(ticket), ctypes.byref(done)))
        return bool(done.value)

    def resample_poly(self, x, up: int, down: int, taps) -> numpy.ndarray:
        """scipy.signal.resample_poly's filtering step on the device (wave_io.resample designs `taps`)."""
        x = _f32(x)
        taps = numpy.ascontiguousarray(taps, dtype=numpy.float64)
        n = self.lib.ryk_resample_length(len(x), int(up), int(down))
        y = numpy.empty(max(n, 1), dtype=numpy.float32)
        no = ctypes.c_int()
        self._check(self.lib.ryk_resample_poly(self._h, _fp(x), len(x), int(up), int(down), _dp(taps), len(taps), _fp(y), len(y), ctypes.byref(no)))
        return y[:no.value]

    F0_METHODS = {'dio': 0, 'harvest': 1, 'crepe': 2}

    def set_f0_method(self, method: str):
        """f0 extractor of world_f0 / world_analyze / sessions created afterwards: 'dio' (pyworld.dio + stonemask, default),
        'harvest' (pyworld.harvest + stonemask) -- yukarin's AcousticFeature.extract f0 hook (acoustic_feature_wrapper.py:28-33) --
        or 'crepe' (sessions only; needs a loaded CREPE model, realtime_yukarin_b200.crepe.load_crepe_model)."""
        self._check(self.lib.ryk_engine_set_f0_method(self._h, self.F0_METHODS[method]))

    @property
    def f0_method(self) -> str:
        return ['dio', 'harvest', 'crepe'][self.lib.ryk_engine_get_f0_method(self._h)]

    def debug_harvest(self, n, fs, frame_period, f0_floor, f0_ceil):
        """Intermediate arrays of the last Harvest analysis with this plan (see ryk_debug_harvest)."""
        import math
        ratio = int(fs / 8000.0 + 0.5)
        channels = 1 + int(math.log((f0_ceil * 1.1) / (f0_floor * 0.9)) / 0.69314718055994529 * 40.0)
        nf1 = int(1000.0 * n / fs) + 1
        ylen = -(-n // ratio)
        maxc = int(channels / 10.0 + 0.5) * 7
        info = numpy.zeros(7, numpy.int32)
        out = dict(y=numpy.zeros(ylen), raw=numpy.zeros((channels, nf1)), cand=numpy.zeros((nf1, maxc)), score=numpy.zeros((nf1, maxc)),
                   best=numpy.zeros(nf1), basic=numpy.zeros(nf1), f0_raw=numpy.zeros(dio_num_frames(fs, n, frame_period)))
        self._check(self.lib.ryk_debug_harvest(self._h, int(n), int(fs), ctypes.c_double(frame_period), ctypes.c_double(f0_floor),
                                               ctypes.c_double(f0_ceil), info.ctypes.data_as(c_int_p), _dp(out['y']), _dp(out['raw']),
                                               _dp(out['cand']), _dp(out['score']), _dp(out['best']), _dp(out['basic']), _dp(out['f0_raw'])))
        assert (info[0], info[1], info[2], info[4]) == (channels, nf1, ylen, maxc), info
        out['nc'] = int(info[6])
        return out

    def test_conv_layer(self, in0, in1, W, scale, shift, transposed, k, stride, pad, act, use_tc, repeat=0):
        """One conv layer in isolation; in0/in1 NHWC float32, W in the Chainer layout. Returns (out NHWC, ms per run)."""
        in0 = _f32(in0)
        B, H, Wd, C0 = in0.shape
        C1 = 0 if in1 is None else in1.shape[3]
        in1a = _f32(in1) if in1 is not None else numpy.zeros(1, numpy.float32)
        W, scale, shift = _f32(W), _f32(scale), _f32(shift)
        cout = W.shape[1] if transposed else W.shape[0]
        if H == 1:
            Ho = 1
        else:
            Ho = (H - 1) * stride + k - 2 * pad if transposed else (H + 2 * pad - k) // stride + 1
        Wo = (Wd - 1) * stride + k - 2 * pad if transposed else (Wd + 2 * pad - k) // stride + 1
        out = numpy.empty((B, Ho, Wo, cout), numpy.float32)
        ms = ctypes.c_float()
        self._check(self.lib.ryk_test_conv_layer(
            self._h, int(transposed), int(k), int(stride), int(pad), B, H, Wd, C0, C1, cout, _fp(in0), _fp(in1a), _fp(W),
            _fp(scale), _fp(shift), int(act), int(use_tc), int(repeat), _fp(out), ctypes.byref(ms)))
        return out, ms.value

    def test_stage2_forward(self, x, keep=(), mode=0, tw=0):
        """One stage-2 forward on NaN-filled buffers (ryk_test_stage2_forward); x [B][Tp][512] float32, keep = [(begin, len), ...];
        mode 3 skips the padded tail from row tw on.  Returns y [B][Tp][512]; rows the plan does not compute stay NaN."""
        x = _f32(x)
        B, Tp, W = x.shape
        assert W == 512
        kb = numpy.array([k[0] for k in keep] or [0], numpy.int32)
        kl = numpy.array([k[1] for k in keep] or [0], numpy.int32)
        y = numpy.empty_like(x)
        self._check(self.lib.ryk_test_stage2_forward(self._h, B, Tp, len(keep), kb.ctypes.data_as(c_int_p), kl.ctypes.data_as(c_int_p),
                                                     int(mode), int(tw), _fp(x), _fp(y)))
        return y

    # ---- sessions ----
    def session_create(self, cfg: SessionConfig, voice: int = 0) -> int:
        sid = ctypes.c_int()
        if voice == 0:
            self._check(self.lib.ryk_session_create(self._h, ctypes.byref(cfg), ctypes.byref(sid)))
        else:
            self._check(self.lib.ryk_session_create_voice(self._h, ctypes.byref(cfg), int(voice), ctypes.byref(sid)))
        self._session_fs[sid.value] = int(cfg.fs)
        return sid.value

    def _session_set_rate(self, fn, sid: int, rate: int, rate_from: int, rate_to: int):
        from .wave_io import resample_filter
        g = math.gcd(int(rate_from), int(rate_to))
        up, down = int(rate_to) // g, int(rate_from) // g
        taps = numpy.ascontiguousarray(resample_filter(up, down), dtype=numpy.float64)
        self._check(fn(self._h, sid, int(rate), up, down, _dp(taps), len(taps)))

    def session_set_input_rate(self, sid: int, rate: int):
        """Take this fresh session's chunks at `rate` (round(rate * buffer_time) samples each), resampled to the session's rate on the
        device with wave_io.resample_filter.  rate == the session's rate: nothing to do."""
        fs = self._session_fs[sid]
        self._session_set_rate(self.lib.ryk_session_set_input_rate, sid, rate, rate, fs)

    def session_set_output_rate(self, sid: int, rate: int):
        """Return this fresh session's samples at `rate`, resampled from the session's rate on the device."""
        fs = self._session_fs[sid]
        self._session_set_rate(self.lib.ryk_session_set_output_rate, sid, rate, fs, rate)

    def session_io_geometry(self, sid: int) -> Dict[str, int]:
        """n_in (samples per chunk), max_out (most samples one step returns), delay_in (input delay, model-rate samples), in_rate,
        out_rate (device rates; the session's rate when unset)."""
        v = [ctypes.c_int() for _ in range(5)]
        self._check(self.lib.ryk_session_io_geometry(self._h, sid, *[ctypes.byref(x) for x in v]))
        return dict(zip(('n_in', 'max_out', 'delay_in', 'in_rate', 'out_rate'), (x.value for x in v)))

    # ---- the session's f0 map and the log-f0 statistics of its speaker ----
    def session_get_f0_map(self, sid: int) -> Dict[str, float]:
        """in_mean, in_std, target_mean, target_std that the next submitted step of the session uses (in follow mode the input side is
        the fallback)."""
        m = F0Map()
        self._check(self.lib.ryk_session_get_f0_map(self._h, sid, ctypes.byref(m)))
        return {k: getattr(m, k) for k in F0Map.KEYS}

    def session_set_f0_map(self, sid: int, in_mean=None, in_std=None, target_mean=None, target_std=None, semitones: float = 0.0):
        """Change this session's f0 map from its next submitted step on (chunks in flight keep theirs; other sessions of the voice are
        not affected).  None keeps the current value.  `semitones` adds semitones * ln(2) / 12 to the target mean (the one given, else
        the current one): that is the whole pitch control -- f0 moves, the spectral envelope (the formants) does not."""
        new = updated_f0_map(self.session_get_f0_map(sid), in_mean, in_std, target_mean, target_std, semitones)
        m = F0Map(*[new[k] for k in F0Map.KEYS])
        self._check(self.lib.ryk_session_set_f0_map(self._h, sid, ctypes.byref(m)))

    def session_f0_measure(self, sid: int, enable: bool = True):
        """Fresh session only: keep running statistics of ln f0 over the voiced frames of the session's input on the device."""
        self._check(self.lib.ryk_session_f0_measure(self._h, sid, int(bool(enable))))

    def session_f0_follow(self, sid: int, follow: bool = True, min_voiced_frames: int = 200, sd_floor: float = F0_SD_FLOOR):
        """Needs session_f0_measure.  From the next submitted step on, a step whose count of voiced frames has reached
        `min_voiced_frames` (200 frames = 1 s of voiced speech) converts with the measured mean and max(measured std, sd_floor) as the
        input side of its f0 map; follow=False returns to the values set from the host."""
        self._check(self.lib.ryk_session_f0_follow(self._h, sid, int(bool(follow)), int(min_voiced_frames), ctypes.c_double(sd_floor)))

    def session_f0_measure_reset(self, sid: int):
        """The statistics restart from zero at the next submitted step."""
        self._check(self.lib.ryk_session_f0_measure_reset(self._h, sid))

    def session_f0_measured(self, sid: int):
        """(voiced frames counted, mean, standard deviation) of ln f0 over the submitted steps (waits for their stage 1)."""
        n, mean, std = ctypes.c_longlong(), ctypes.c_double(), ctypes.c_double()
        self._check(self.lib.ryk_session_f0_measured(self._h, sid, ctypes.byref(n), ctypes.byref(mean), ctypes.byref(std)))
        return n.value, mean.value, std.value

    def session_destroy(self, sid: int):
        self._check(self.lib.ryk_session_destroy(self._h, sid))
        self._session_fs.pop(sid, None)

    def session_push(self, sid: int, wave, out: Optional[numpy.ndarray] = None) -> numpy.ndarray:
        w = _f32(wave)
        if out is None:
            out = numpy.empty(max(len(w) * 2 + 8192, self.session_io_geometry(sid)['max_out']), dtype=numpy.float64)
        n_out = ctypes.c_int()
        self._check(self.lib.ryk_session_push(self._h, sid, _fp(w), len(w), _dp(out), len(out), ctypes.byref(n_out)))
        return out[:n_out.value]

    def session_submit(self, sid: int, wave) -> int:
        w = _f32(wave)
        ticket = ctypes.c_longlong()
        self._check(self.lib.ryk_session_submit(self._h, sid, _fp(w), len(w), ctypes.byref(ticket)))
        return ticket.value

    def session_collect(self, sid: int, ticket: int, out: numpy.ndarray) -> numpy.ndarray:
        n_out = ctypes.c_int()
        self._check(self.lib.ryk_session_collect(self._h, sid, ctypes.c_longlong(ticket), _dp(out), len(out), ctypes.byref(n_out)))
        return out[:n_out.value]

    def session_poll(self, sid: int, ticket: int) -> bool:
        """True when session_collect(ticket) would return without waiting (cudaEventQuery, never blocks)."""
        done = ctypes.c_int()
        self._check(self.lib.ryk_session_poll(self._h, sid, ctypes.c_longlong(ticket), ctypes.byref(done)))
        return bool(done.value)

    def session_push_device(self, sid: int, wave_dev_ptr: int, n: int, out_dev_ptr: int, out_capacity: int, n_out_dev_ptr: int):
        self._check(self.lib.ryk_session_push_device(self._h, sid, ctypes.c_void_p(wave_dev_ptr), int(n), ctypes.c_void_p(out_dev_ptr),
                                                     int(out_capacity), ctypes.c_void_p(n_out_dev_ptr)))

    def session_stage_times(self, sid: int):
        """(start, end) arrays of shape (steps, 5) in ms; see ryk_session_stage_times."""
        st, en = (ctypes.c_float * 40)(), (ctypes.c_float * 40)()
        n = self._check(self.lib.ryk_session_stage_times(self._h, sid, st, en))
        return numpy.array(st[:n * 5]).reshape(n, 5), numpy.array(en[:n * 5]).reshape(n, 5)

    # ---- groups (several streams per GPU, one batched stage-2 forward per step) ----
    def group_create(self, session_ids: Sequence[int]) -> int:
        ids = (ctypes.c_int * len(session_ids))(*[int(i) for i in session_ids])
        gid = ctypes.c_int()
        self._check(self.lib.ryk_group_create(self._h, ids, len(session_ids), ctypes.byref(gid)))
        return gid.value

    def group_destroy(self, gid: int):
        self._check(self.lib.ryk_group_destroy(self._h, gid))

    def group_size(self, gid: int) -> int:
        return self._check(self.lib.ryk_group_size(self._h, gid))

    def group_add(self, gid: int, sid: int):
        """Make session `sid` (fresh or running, in no group, nothing uncollected) the group's last member between two steps; its
        stream continues where it was."""
        self._check(self.lib.ryk_group_add(self._h, gid, int(sid)))

    def group_remove(self, gid: int, sid: int):
        """Take member `sid` out of the group between two steps (the members after it move down one slot); it continues as an
        ungrouped session."""
        self._check(self.lib.ryk_group_remove(self._h, gid, int(sid)))

    def group_members(self, gid: int) -> List[int]:
        """Member session ids in slot order: the order of the waves / outputs of group_submit, group_collect and group_push_device."""
        n = self._check(self.lib.ryk_group_members(self._h, gid, None, 0))
        ids = (ctypes.c_int * max(n, 1))()
        n = self._check(self.lib.ryk_group_members(self._h, gid, ids, n))
        return [int(ids[i]) for i in range(n)]

    def group_submit(self, gid: int, waves: Sequence) -> int:
        ws = [_f32(w) for w in waves]
        ptrs = (ctypes.POINTER(ctypes.c_float) * len(ws))(*[_fp(w) for w in ws])
        ticket = ctypes.c_longlong()
        self._check(self.lib.ryk_group_submit(self._h, gid, ptrs, len(ws[0]), ctypes.byref(ticket)))
        return ticket.value

    def group_collect(self, gid: int, ticket: int, outs: Sequence[numpy.ndarray]) -> List[numpy.ndarray]:
        ptrs = (ctypes.POINTER(ctypes.c_double) * len(outs))(*[_dp(o) for o in outs])
        n_outs = (ctypes.c_int * len(outs))()
        self._check(self.lib.ryk_group_collect(self._h, gid, ctypes.c_longlong(ticket), ptrs, min(len(o) for o in outs), n_outs))
        return [o[:n] for o, n in zip(outs, n_outs)]

    def group_push_device(self, gid: int, wave_dev_ptrs: Sequence[int], n: int, out_dev_ptrs: Sequence[int], out_capacity: int,
                          n_out_dev_ptrs: Sequence[int]):
        B = len(wave_dev_ptrs)
        w = (ctypes.c_void_p * B)(*[int(p) for p in wave_dev_ptrs])
        o = (ctypes.c_void_p * B)(*[int(p) for p in out_dev_ptrs])
        c = (ctypes.c_void_p * B)(*[int(p) for p in n_out_dev_ptrs])
        self._check(self.lib.ryk_group_push_device(self._h, gid, w, int(n), o, int(out_capacity), c))



_default: Optional[Engine] = None


def default_engine() -> Engine:
    """Process-wide engine on cuda:LOCAL_RANK (created on first use)."""
    global _default
    if _default is None:
        _default = Engine()
    return _default


def set_default_engine(engine: Optional[Engine]):
    global _default
    _default = engine
