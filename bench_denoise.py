"""Cost of the input noise suppression on the headline stream: steps per second of one device-resident session
(ryk_session_push_device, precision 1, 0.3 s chunks at 24 kHz, extras 0 / 0.5 / 0, full-width synthetic voice) in three variants:

  off      the session without the filter
  profile  ryk_session_denoise with a noise profile set before the first step (reduction 20 dB)
  learn    ryk_session_denoise learning a profile on every step (one learning longer than the run)

Each variant is a session of its own on one engine, created with RYK_STAGE_TIMES=1.  A leg queues --steps steps in blocks of --block
(the device drains between blocks, as in bench.py's sustained figure) and is timed on the host clock from an idle device to an idle
device; the legs of the variants alternate within each of --repeats rounds, after --warmup steps per session.  Reported per variant:
every round's steps/s and their median, the kernels per step from ryk_engine_launch_count, and the median device time of the gate stage
(input resampler, filter, wave slides) over the last 8 steps of every leg.  The card's name and power limit are recorded with the numbers.

    python bench_denoise.py [--out DIR] [--steps 3000 --block 100 --warmup 40 --repeats 3]

Prints one JSON line (and writes it to DIR/bench_denoise.json with --out).  Needs a CUDA device; there is no CPU path."""
import argparse
import json
import os
import shutil
import statistics
import tempfile
import time
from pathlib import Path

import numpy as np

from bench_f0_control import EXTRA, FS, T, card

VARIANTS = ('off', 'profile', 'learn')


def make_parser():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', type=Path, default=None)
    ap.add_argument('--steps', type=int, default=3000)
    ap.add_argument('--block', type=int, default=100)
    ap.add_argument('--warmup', type=int, default=40)
    ap.add_argument('--repeats', type=int, default=3)
    return ap


def main(argv=None):
    args = make_parser().parse_args(argv)
    import torch
    if not torch.cuda.is_available():
        raise SystemExit('bench_denoise.py needs a CUDA device')
    from realtime_yukarin_b200 import synthetic
    from realtime_yukarin_b200.engine import Engine, SessionConfig
    from realtime_yukarin_b200.models import load_voice

    tmp = Path(tempfile.mkdtemp(prefix='bench_denoise_'))           # synthetic model files: never written into the tree
    eng = Engine()
    eng.set_precision('fp16')
    paths = synthetic.write_synthetic_models(tmp / 'v0', seed=0)
    voice = eng.voice_create()
    load_voice(eng, voice, **{k: paths[k] for k in ('stage1_model_path', 'stage2_model_path', 'input_statistics_path', 'target_statistics_path')})
    cfg = SessionConfig(fs=FS, frame_period_ms=5.0, f0_floor=71.0, f0_ceil=800.0, fft_length=1024, order=8, alpha=0.466, buffer_time=T,
                        encode_extra_time=EXTRA[0], convert_extra_time=EXTRA[1], decode_extra_time=EXTRA[2], threshold_db=60.0,
                        vocoder_buffer_size=1024)
    n = round(T * FS)
    n_chunks = 64
    x = synthetic.synthetic_speech((n_chunks + 1) * T, stream=0)
    x = (x + 0.01 * np.random.default_rng(0).standard_normal(len(x))).astype(np.float32)
    d_in = torch.from_numpy(np.stack([x[k * n:(k + 1) * n] for k in range(n_chunks)])).cuda()
    prev = os.environ.get('RYK_STAGE_TIMES')
    os.environ['RYK_STAGE_TIMES'] = '1'
    try:
        sids = {v: eng.session_create(cfg, voice=voice) for v in VARIANTS}
    finally:
        if prev is None:
            os.environ.pop('RYK_STAGE_TIMES', None)
        else:
            os.environ['RYK_STAGE_TIMES'] = prev
    for v in ('profile', 'learn'):
        eng.session_denoise(sids[v])
    eng.session_set_noise_profile(sids['profile'], np.full(257, 0.01 ** 2 * 256.0))    # white noise at 0.01 RMS: sum(w^2) = 256
    eng.session_denoise_learn(sids['learn'], frames=10 ** 12)
    cap = eng.session_io_geometry(sids['off'])['max_out']
    ring = 8                                      # distinct output slots: consecutive steps are in flight together
    d_out = torch.empty((ring, cap), dtype=torch.float64, device='cuda')
    d_n = torch.zeros((ring, 1), dtype=torch.int32, device='cuda')
    step_no = {v: 0 for v in VARIANTS}

    def push(v):
        k = step_no[v]
        eng.session_push_device(sids[v], d_in[k % n_chunks].data_ptr(), n, d_out[k % ring].data_ptr(), cap, d_n[k % ring].data_ptr())
        step_no[v] = k + 1

    def leg(v, steps):
        eng.synchronize()
        launches0 = eng.launch_count
        t0 = time.perf_counter()
        done = 0
        while done < steps:
            for _ in range(min(args.block, steps - done)):
                push(v)
            done += min(args.block, steps - done)
            eng.synchronize()
        s = time.perf_counter() - t0
        start, end = eng.session_stage_times(sids[v])
        return steps / s, (eng.launch_count - launches0) / steps, float(np.median(end[:, 0] - start[:, 0]))

    for v in VARIANTS:
        leg(v, args.warmup)
    rates = {v: [] for v in VARIANTS}
    gate = {v: [] for v in VARIANTS}
    kernels = {}
    for _ in range(args.repeats):
        for v in VARIANTS:
            r, kernels[v], g = leg(v, args.steps)
            rates[v].append(r)
            gate[v].append(g)
    left = eng.session_noise_profile(sids['learn'])[1]
    for sid in sids.values():
        eng.session_destroy(sid)
    eng.voice_destroy(voice)
    shutil.rmtree(tmp, ignore_errors=True)
    line = dict(card=card(), buffer_time=T, extras=EXTRA, steps=args.steps, block=args.block, warmup=args.warmup, repeats=args.repeats,
                learn_frames_left=left,
                variants={v: dict(steps_per_s=statistics.median(rates[v]), steps_per_s_all=rates[v], kernels_per_step=kernels[v],
                                  gate_ms=statistics.median(gate[v]), gate_ms_all=gate[v])
                          for v in VARIANTS})
    if args.out is not None:
        args.out.mkdir(parents=True, exist_ok=True)
        (args.out / 'bench_denoise.json').write_text(json.dumps(line, indent=1))
    print(json.dumps(line))


if __name__ == '__main__':
    main()
