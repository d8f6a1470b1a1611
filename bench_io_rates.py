"""Cost of running a streaming session at a sound card's rates (device-side resampling into and out of the session).

Legs, each one 1-stream session at 0.3 s chunks (extras 0 / 0.5 / 0, full-width synthetic U-Nets, precision 1) with device rates
in/out of 24/24 kHz (no resampler, the reference point), 48/48, 44.1/44.1 and 48/24 kHz, plus a 4-stream group at 48/48 kHz.  Each leg
creates its sessions, warms up their graphs, then times --steps device-resident steps with CUDA events on the engine's stopwatch; the
legs alternate over --rounds rounds so that clock and neighbour drift spreads over all of them.  Reported per leg: ms per step and
chunks/s (median over rounds; a group step is one chunk per member).  With RYK_STAGE_TIMES=1 in the environment it also reports the
device time of the gate stage (input resampling + wave slides + silence gate) and of the synthesis stage (synthesizer + output
resampling), mean over the last 8 steps of the first session.  The card's name and power limit are recorded with the numbers.

    python bench_io_rates.py --out DIR [--steps 200 --warmup 20 --rounds 3]

Writes DIR/bench_io_rates.json and prints it.  Needs a CUDA device; there is no CPU path."""
import argparse
import json
import os
import shutil
import statistics
import subprocess
import tempfile
from pathlib import Path

import numpy as np

T, EXTRA, FS = 0.3, (0.0, 0.5, 0.0), 24000
LEGS = [(24000, 24000, 1), (48000, 48000, 1), (44100, 44100, 1), (48000, 24000, 1), (48000, 48000, 4)]


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else 'unknown (nvidia-smi unavailable)'


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', type=Path, required=True)
    ap.add_argument('--steps', type=int, default=200)
    ap.add_argument('--warmup', type=int, default=20)
    ap.add_argument('--rounds', type=int, default=3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit('bench_io_rates.py needs a CUDA device')
    stage_times = os.environ.get('RYK_STAGE_TIMES', '0') not in ('', '0')
    from realtime_yukarin_b200 import synthetic, wave_io
    from realtime_yukarin_b200.engine import Engine, SessionConfig
    from realtime_yukarin_b200.models import AcousticConverter, F0Converter, SuperResolution
    from realtime_yukarin_b200.params import create_from_json, create_sr_from_json

    tmp = Path(tempfile.mkdtemp(prefix='bench_io_rates_'))    # synthetic model files: never written into the tree
    paths = synthetic.write_synthetic_models(tmp, seed=0)
    eng = Engine()
    f0c = F0Converter(paths['input_statistics_path'], paths['target_statistics_path'])
    AcousticConverter(create_from_json(paths['stage1_config_path']), paths['stage1_model_path'], f0_converter=f0c, engine=eng)
    SuperResolution(create_sr_from_json(paths['stage2_config_path']), paths['stage2_model_path'], engine=eng)
    eng.set_precision('fp16')
    total = args.warmup + args.steps
    x24 = synthetic.synthetic_speech((total + 1) * T, stream=0)
    inputs = {}                                       # device rate -> (total, n_in) chunks on the device
    for rate in sorted({leg[0] for leg in LEGS}):
        n_in = round(T * rate)
        x = wave_io.resample(x24, FS, rate, eng)
        inputs[rate] = torch.from_numpy(np.stack([x[k * n_in:(k + 1) * n_in] for k in range(total)])).cuda()
    cfg = SessionConfig(fs=FS, frame_period_ms=5.0, f0_floor=71.0, f0_ceil=800.0, fft_length=1024, order=8, alpha=0.466, buffer_time=T,
                        encode_extra_time=EXTRA[0], convert_extra_time=EXTRA[1], decode_extra_time=EXTRA[2], threshold_db=60.0,
                        vocoder_buffer_size=1024)

    def leg(rate_in, rate_out, members):
        sids = []
        for _ in range(members):
            sid = eng.session_create(cfg)
            eng.session_set_input_rate(sid, rate_in)
            eng.session_set_output_rate(sid, rate_out)
            sids.append(sid)
        g = eng.session_io_geometry(sids[0])
        d_in = inputs[rate_in]
        d_out = torch.empty((members, 8, g['max_out']), dtype=torch.float64, device='cuda')
        d_n = torch.zeros((members, 8), dtype=torch.int32, device='cuda')
        gid = eng.group_create(sids) if members > 1 else None

        def push(k):
            if gid is None:
                eng.session_push_device(sids[0], d_in[k].data_ptr(), g['n_in'], d_out[0, k % 8].data_ptr(), g['max_out'], d_n[0, k % 8:].data_ptr())
            else:
                eng.group_push_device(gid, [d_in[k].data_ptr()] * members, g['n_in'], [d_out[i, k % 8].data_ptr() for i in range(members)],
                                      g['max_out'], [d_n[i, k % 8:].data_ptr() for i in range(members)])
        for k in range(args.warmup):
            push(k)
        eng.synchronize()
        eng.timer_start()
        for k in range(args.warmup, total):
            push(k)
        ms = eng.timer_stop()
        gate = synth = None
        if stage_times:
            st, en = eng.session_stage_times(sids[0])
            gate, synth = float((en[:, 0] - st[:, 0]).mean()), float((en[:, 4] - st[:, 4]).mean())
        if gid is not None:
            eng.group_destroy(gid)
        for sid in sids:
            eng.session_destroy(sid)
        return ms / args.steps, gate, synth

    results = {leg_: [] for leg_ in LEGS}
    leg(*LEGS[-1])                                   # first-use costs (module load, cuFFT plans, group plan) outside the rounds
    for _ in range(args.rounds):
        for leg_ in LEGS:
            results[leg_].append(leg(*leg_))
    rows = []
    for (rate_in, rate_out, members), v in results.items():
        ms = statistics.median(a for a, _, _ in v)
        row = dict(rate_in=rate_in, rate_out=rate_out, streams=members, ms_per_step=ms, chunks_per_s=members * 1000.0 / ms,
                   ms_per_step_all=[a for a, _, _ in v])
        if stage_times:
            row.update(gate_stage_ms=statistics.median(b for _, b, _ in v), synth_stage_ms=statistics.median(c for _, _, c in v))
        rows.append(row)
    line = dict(card=card(), buffer_time=T, extras=EXTRA, steps=args.steps, warmup=args.warmup, rounds=args.rounds, stage_times=stage_times,
                legs=rows)
    shutil.rmtree(tmp, ignore_errors=True)
    args.out.mkdir(parents=True, exist_ok=True)
    (args.out / 'bench_io_rates.json').write_text(json.dumps(line, indent=1))
    print(json.dumps(line))


if __name__ == '__main__':
    main()
