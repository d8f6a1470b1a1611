"""ryk_engine_launch_count against an independent count: the CUDA kernels torch.profiler (CUPTI) sees while session and group steps
run, which include the kernels inside the stage graphs and the stage-1 SWITCH bodies.  Each window starts at a fresh session, so it
covers the first (capturing) launch of every stage graph and the synthesizer's noise top-up.  No torch CUDA work runs inside a window:
every kernel in it belongs to the steps."""
import json
import os
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

from realtime_yukarin_b200 import synthetic
from realtime_yukarin_b200.engine import SessionConfig

from .test_gpu_parity import _load

pytestmark = pytest.mark.gpu

FS, T = 24000, 0.3
STEPS = 20


def _cfg():
    return SessionConfig(fs=FS, frame_period_ms=5.0, f0_floor=71.0, f0_ceil=800.0, fft_length=1024, order=8, alpha=0.466, buffer_time=T,
                         encode_extra_time=0.0, convert_extra_time=0.5, decode_extra_time=0.0, threshold_db=60.0, vocoder_buffer_size=1024)


def _speech(steps, stream, rate=FS):
    n = round(T * rate)
    x = synthetic.synthetic_speech((steps + 1) * T, stream=stream, fs=rate)
    return [np.ascontiguousarray(x[k * n:(k + 1) * n]) for k in range(steps)]


def _kernel_events(prof, path):
    """the CUDA kernel events of a finished torch.profiler window, read back from the chrome trace it writes to path"""
    prof.export_chrome_trace(str(path))
    ev = json.loads(path.read_text())
    ev = ev['traceEvents'] if isinstance(ev, dict) else ev
    return [e for e in ev if e.get('cat') == 'kernel' and e.get('ph') == 'X']


def _window(engine, tmp_path, run):
    """(CUDA kernels the profiler saw, change of engine.launch_count) over run()"""
    from torch.profiler import ProfilerActivity, profile
    before = engine.launch_count                         # synchronises the device
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        run()
        engine.synchronize()
    counted = engine.launch_count - before
    return len(_kernel_events(prof, tmp_path / 'trace.json')), counted


def _run_child(tmp_path, module, function):
    """function(tmp_path) of tests/<module>.py run in a Python process of its own; returns what it returned, through JSON.

    Tests that profile outside this module do it this way: CUPTI's teardown and re-initialisation between profiling sessions is not
    reliable in a process that runs CUDA graphs (torch's profiler says as much), and this module's tests expect to be the first
    profiling in their process."""
    root = Path(__file__).resolve().parent.parent
    flags = ['-s'] if sys.flags.no_user_site else []
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([str(root)] + [p for p in [os.environ.get('PYTHONPATH')] if p]))
    out = tmp_path / 'result.json'
    code = (f'import json, pathlib; from tests.{module} import {function}; '
            f'pathlib.Path({str(out)!r}).write_text(json.dumps({function}(pathlib.Path({str(tmp_path)!r}))))')
    subprocess.run([sys.executable, *flags, '-c', code], cwd=root, env=env, check=True, timeout=900)
    return json.loads(out.read_text())


def _session_window(engine, tmp_path, chunks, in_rate=None, out_rate=None, f0_method='dio'):
    """profiled window over the steps of one fresh session fed `chunks` through the host API"""
    prev = engine.f0_method
    engine.set_f0_method(f0_method)
    try:
        sid = engine.session_create(_cfg())
    finally:
        engine.set_f0_method(prev)
    if in_rate:
        engine.session_set_input_rate(sid, in_rate)
    if out_rate:
        engine.session_set_output_rate(sid, out_rate)
    buf = np.empty(engine.session_io_geometry(sid)['max_out'])
    try:
        return _window(engine, tmp_path, lambda: [engine.session_push(sid, c, buf) for c in chunks])
    finally:
        engine.session_destroy(sid)


def _check(name, seen, counted, steps):
    print(f'{name}: {counted} kernels counted, {seen} seen by the profiler over {steps} steps')
    assert counted == seen, (name, counted, seen)


def test_headline_and_layered_stage1(engine, full_models, tmp_path):
    """The headline session (DIO, FP16, fused stage 1) and the same session with stage 1 as the 16-layer sequence; the fused kernel
    runs fewer kernels per step."""
    _load(engine, full_models)
    engine.set_precision('fp16')
    chunks = _speech(STEPS, stream=0)
    per_step = {}
    try:
        for fused in (True, False):
            engine.set_stage1_fused(fused)
            seen, counted = _session_window(engine, tmp_path, chunks)
            _check(f'stage 1 {"fused" if fused else "layered"}', seen, counted, STEPS)
            per_step[fused] = counted / STEPS
    finally:
        engine.set_stage1_fused(True)
    assert per_step[True] < per_step[False], per_step


def test_harvest(engine, full_models, tmp_path):
    _load(engine, full_models)
    engine.set_precision('fp16')
    seen, counted = _session_window(engine, tmp_path, _speech(STEPS, stream=1), f0_method='harvest')
    _check('harvest', seen, counted, STEPS)


def test_crepe(engine, full_models, tmp_path):
    from realtime_yukarin_b200 import crepe as pcrepe
    _load(engine, full_models)
    pcrepe.load_crepe_model(synthetic.write_crepe_model(tmp_path / 'crepe', seed=5, capacity='tiny'), engine)
    engine.set_precision('fp16')
    seen, counted = _session_window(engine, tmp_path, _speech(STEPS, stream=2), f0_method='crepe')
    _check('crepe', seen, counted, STEPS)


@pytest.mark.parametrize('rate', [48000, 44100])
def test_device_rates(engine, full_models, tmp_path, rate):
    _load(engine, full_models)
    engine.set_precision('fp16')
    seen, counted = _session_window(engine, tmp_path, _speech(STEPS, stream=3, rate=rate), in_rate=rate, out_rate=rate)
    _check(f'{rate} Hz in and out', seen, counted, STEPS)


def test_group(engine, full_models, tmp_path):
    _load(engine, full_models)
    engine.set_precision('fp16')
    members = 4
    xs = [_speech(STEPS, stream=10 + j) for j in range(members)]
    sids = [engine.session_create(_cfg()) for _ in range(members)]
    gid = engine.group_create(sids)
    bufs = [np.empty(engine.session_io_geometry(sids[0])['max_out']) for _ in range(members)]

    def run():
        for k in range(STEPS):
            engine.group_collect(gid, engine.group_submit(gid, [x[k] for x in xs]), bufs)
    try:
        seen, counted = _window(engine, tmp_path, run)
    finally:
        engine.group_destroy(gid)
        for sid in sids:
            engine.session_destroy(sid)
    _check(f'group of {members}', seen, counted, STEPS)


@pytest.mark.parametrize('fused', [True, False])
def test_speech_silence_speech(engine, full_models, tmp_path, fused):
    """Speech, then digital silence longer than the convert window, then speech: the stage-1 bucket the device selects changes between
    steps (a window that holds some speech keeps only its loud frames; a window of silence keeps every frame)."""
    _load(engine, full_models)
    engine.set_precision('fp16')
    n = round(T * FS)
    speech = _speech(14, stream=4)
    chunks = speech[:6] + [np.zeros(n, np.float32)] * 12 + speech[6:]
    try:
        engine.set_stage1_fused(fused)
        seen, counted = _session_window(engine, tmp_path, chunks)
    finally:
        engine.set_stage1_fused(True)
    _check(f'speech / silence / speech, stage 1 {"fused" if fused else "layered"}', seen, counted, len(chunks))
