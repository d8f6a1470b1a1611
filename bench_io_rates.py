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
import os
import shutil
import statistics
import tempfile
from pathlib import Path

from benchlib import (EXTRA, FS, T, bench_parser, card, device_chunks, device_pusher, emit, headline_config, require_cuda, stopwatch_ms,
                      synthetic_builtin)

LEGS = [(24000, 24000, 1), (48000, 48000, 1), (44100, 44100, 1), (48000, 24000, 1), (48000, 48000, 4)]


def main():
    args = bench_parser(required_out=True, steps=200, warmup=20, rounds=3).parse_args()
    require_cuda('bench_io_rates.py')
    stage_times = os.environ.get('RYK_STAGE_TIMES', '0') not in ('', '0')
    from realtime_yukarin_b200 import synthetic, wave_io
    from realtime_yukarin_b200.engine import Engine

    tmp = Path(tempfile.mkdtemp(prefix='bench_io_rates_'))    # synthetic model files: never written into the tree
    eng = Engine()
    synthetic_builtin(eng, tmp)
    eng.set_precision('fp16')
    total = args.warmup + args.steps
    x24 = synthetic.synthetic_speech((total + 1) * T, stream=0)
    inputs = {}                                       # device rate -> (total, n_in) chunks on the device
    for rate in sorted({leg[0] for leg in LEGS}):
        inputs[rate] = device_chunks(wave_io.resample(x24, FS, rate, eng), round(T * rate), total)
    cfg = headline_config()

    def leg(rate_in, rate_out, members):
        sids = []
        for _ in range(members):
            sid = eng.session_create(cfg)
            eng.session_set_input_rate(sid, rate_in)
            eng.session_set_output_rate(sid, rate_out)
            sids.append(sid)
        push = device_pusher(eng, inputs[rate_in], eng.session_io_geometry(sids[0])['max_out'], members)
        gid = eng.group_create(sids) if members > 1 else None
        ms = stopwatch_ms(eng, (lambda: push(sids[0])) if gid is None else (lambda: push(gid, group=True)), args.warmup, args.steps)
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
    emit(args.out, 'bench_io_rates', line)


if __name__ == '__main__':
    main()
