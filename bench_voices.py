"""Cost of mixing target voices in one group: the batched stage-2 forward reads each member's weights from its own voice.

Legs: a device-resident group (ryk_group_push_device, precision 1, extras 0 / 0.5 / 0) of 8 members at 1.0 s chunks (BASELINE config 5
shape, Tp 512) and of 4 members at 0.3 s chunks, with 1, 2, 4 and (8 members only) 8 distinct voices (member i converts into voice
i mod V; the voices are full-width synthetic models of seeds 0..7).  Each leg creates its sessions and group, warms up its graphs, times --steps
steps on the engine's device stopwatch (profiling off), then runs --steps more with stage-2 event timing (ryk_engine_profile) for the
device time of the batched forward.  Legs alternate over --rounds rounds.  Reported per leg: chunks/s and ms per step (median over
rounds; a step is one chunk per member) and the stage-2 device ms per forward (median).  Also printed, computed from the shapes only:
the stage-2 weight bytes one forward streams at FP16 for V voices.  The card's name and power limit are recorded with the numbers.

    python bench_voices.py [--out DIR] [--steps 60 --warmup 10 --rounds 3]

Prints one JSON line (and writes it to DIR/bench_voices.json with --out).  Needs a CUDA device; there is no CPU path."""
import shutil
import statistics
import tempfile
from pathlib import Path

from benchlib import (EXTRA, FS, bench_parser, card, device_chunks, device_pusher, emit, headline_config, require_cuda, stopwatch_ms,
                      synthetic_voice)

GROUPS = [(8, 1.0), (4, 0.3)]
VOICES = [1, 2, 4, 8]


def stage2_weight_bytes(base=64):
    """FP16 bytes of one voice's stage-2 weights (every layer; the two 3x3 edge layers are a few KB)."""
    from realtime_yukarin_b200.engine import _unet_layer_shapes
    return sum(cin * cout * k * k for _, cin, cout, k in _unet_layer_shapes(2, 1, 1, base)) * 2


def main():
    args = bench_parser(steps=60, warmup=10, rounds=3).parse_args()
    require_cuda('bench_voices.py')
    from realtime_yukarin_b200 import synthetic
    from realtime_yukarin_b200.engine import Engine

    tmp = Path(tempfile.mkdtemp(prefix='bench_voices_'))       # synthetic model files: never written into the tree
    eng = Engine()
    eng.set_precision('fp16')
    voices = [synthetic_voice(eng, tmp, seed) for seed in range(max(VOICES))]
    total = args.warmup + 2 * args.steps
    chunks = {}
    for _, T in GROUPS:
        chunks[T] = device_chunks(synthetic.synthetic_speech((total + 1) * T, stream=0), round(T * FS), total)

    def leg(members, T, n_voices):
        sids = [eng.session_create(headline_config(buffer_time=T), voice=voices[i % n_voices]) for i in range(members)]
        gid = eng.group_create(sids)
        push = device_pusher(eng, chunks[T], eng.session_io_geometry(sids[0])['max_out'], members)
        ms = stopwatch_ms(eng, lambda: push(gid, group=True), args.warmup, args.steps)
        eng.profile_read2()                       # drop events of earlier forwards
        eng.profile(True)
        for _ in range(args.steps):
            push(gid, group=True)
        s2_total, _, runs = eng.profile_read2()
        eng.profile(False)
        eng.group_destroy(gid)
        for sid in sids:
            eng.session_destroy(sid)
        return ms / args.steps, s2_total / max(runs, 1)

    legs = [(m, T, v) for m, T in GROUPS for v in VOICES if v <= m]      # a group of m members holds at most m distinct voices
    results = {leg_: [] for leg_ in legs}
    for m, T in GROUPS:
        leg(m, T, max(VOICES))                    # first-use costs (module load, cuFFT plans, group plans) outside the rounds
    for _ in range(args.rounds):
        for leg_ in legs:
            results[leg_].append(leg(*leg_))
    wb = stage2_weight_bytes()
    rows = []
    for (members, T, n_voices), r in results.items():
        ms = statistics.median(a for a, _ in r)
        rows.append(dict(members=members, buffer_time=T, voices=n_voices, ms_per_step=ms, chunks_per_s=members * 1000.0 / ms,
                         stage2_ms_per_forward=statistics.median(b for _, b in r), ms_per_step_all=[a for a, _ in r],
                         stage2_weight_mb=n_voices * wb / 1e6))
    line = dict(card=card(), extras=EXTRA, steps=args.steps, warmup=args.warmup, rounds=args.rounds, stage2_weight_mb_per_voice=wb / 1e6,
                legs=rows)
    for v in voices:
        eng.voice_destroy(v)
    shutil.rmtree(tmp, ignore_errors=True)
    emit(args.out, 'bench_voices', line)


if __name__ == '__main__':
    main()
