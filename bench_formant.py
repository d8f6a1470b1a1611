"""Cost of the per-session formant ratio on the headline stream: steps per second of one device-resident session
(ryk_session_push_device, precision 1, 0.3 s chunks, extras 0 / 0.5 / 0, full-width synthetic voice) in three variants:

  off    the session as it is without the feature (ratio 1: the stage-2 epilogue takes the unwarped expression)
  fixed  ryk_session_set_formant(1.2) once before the first step: every step's epilogue warps
  set    ryk_session_set_formant before every step, alternating 0.9 / 1.1: one 64-byte copy on stream C per step

Each variant is a session of its own on one engine.  A leg queues --steps steps in blocks of --block (the device drains between
blocks, as in bench.py's sustained figure) and is timed on the host clock from an idle device to an idle device; the legs of the variants
alternate within each of --repeats rounds, after --warmup steps per session.  Reported per variant: every round's steps/s, their median,
and the kernels per step from ryk_engine_launch_count, which must be equal across variants.  The card's name and power limit are
recorded with the numbers.

    python bench_formant.py [--out DIR] [--steps 3000 --block 100 --warmup 40 --repeats 3]

Prints one JSON line (and writes it to DIR/bench_formant.json with --out).  Needs a CUDA device; there is no CPU path."""
import argparse
import json
import shutil
import statistics
import tempfile
import time
from pathlib import Path

import numpy as np

from bench_f0_control import EXTRA, FS, T, card

VARIANTS = ('off', 'fixed', 'set')


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
        raise SystemExit('bench_formant.py needs a CUDA device')
    from realtime_yukarin_b200 import synthetic
    from realtime_yukarin_b200.engine import Engine, SessionConfig
    from realtime_yukarin_b200.models import load_voice

    tmp = Path(tempfile.mkdtemp(prefix='bench_formant_'))           # synthetic model files: never written into the tree
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
    d_in = torch.from_numpy(np.stack([x[k * n:(k + 1) * n] for k in range(n_chunks)])).cuda()
    sids = {v: eng.session_create(cfg, voice=voice) for v in VARIANTS}
    eng.session_set_formant(sids['fixed'], ratio=1.2)
    cap = eng.session_io_geometry(sids['off'])['max_out']
    ring = 8                                      # distinct output slots: consecutive steps are in flight together
    d_out = torch.empty((ring, cap), dtype=torch.float64, device='cuda')
    d_n = torch.zeros((ring, 1), dtype=torch.int32, device='cuda')
    step_no = {v: 0 for v in VARIANTS}

    def push(v):
        k = step_no[v]
        if v == 'set':                            # a different ratio every step, so that every step stages a copy
            eng.session_set_formant(sids[v], ratio=0.9 if k % 2 else 1.1)
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
        return steps / s, (eng.launch_count - launches0) / steps

    for v in VARIANTS:
        leg(v, args.warmup)
    rates = {v: [] for v in VARIANTS}
    kernels = {}
    for _ in range(args.repeats):
        for v in VARIANTS:
            r, kernels[v] = leg(v, args.steps)
            rates[v].append(r)
    for sid in sids.values():
        eng.session_destroy(sid)
    eng.voice_destroy(voice)
    shutil.rmtree(tmp, ignore_errors=True)
    line = dict(card=card(), buffer_time=T, extras=EXTRA, steps=args.steps, block=args.block, warmup=args.warmup, repeats=args.repeats,
                variants={v: dict(steps_per_s=statistics.median(rates[v]), steps_per_s_all=rates[v], kernels_per_step=kernels[v])
                          for v in VARIANTS})
    if args.out is not None:
        args.out.mkdir(parents=True, exist_ok=True)
        (args.out / 'bench_formant.json').write_text(json.dumps(line, indent=1))
    print(json.dumps(line))


if __name__ == '__main__':
    main()
