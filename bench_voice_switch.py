"""Cost of switching a running session to another voice (ryk_session_set_voice) on the headline stream: precision 1, 0.3 s chunks,
extras 0 / 0.5 / 0, full-width (base 64) synthetic voices.

  call      host wall time of ryk_session_set_voice: a session alone (A <-> B) and a member of an 8-session group of voices A and B
            (the member A <-> C), --switches calls each, one step between them.  The call waits for the device, builds the new
            voice's stage-1 plans, six stage-1 graphs (captured and uploaded) and the stage-2 plans (alone: two lane plans; member: the
            group's batched plan), and releases the old ones.
  stream    steps/s of one device-resident session (ryk_session_push_device) that switches A <-> B every 10 steps, against the same
            session never switching; legs of --steps steps alternate, --repeats rounds, timed on the host clock idle to idle.
  latency   host submit -> collect time of blocking steps (ryk_session_push) around a switch every 20 steps: the first three steps after
            the switch (they capture the stage-2 graphs) against the steady steps 5..19 after it; medians over the switches.

    python bench_voice_switch.py [--out DIR] [--switches 24 --steps 400 --repeats 3]

Prints one JSON line (and writes it to DIR/bench_voice_switch.json with --out).  Needs a CUDA device; there is no CPU path."""
import shutil
import statistics
import tempfile
import time
from pathlib import Path

import numpy as np

from benchlib import (EXTRA, FS, RING, T, alternate, bench_parser, card, device_chunks, emit, headline_config, output_ring,
                      require_cuda, synthetic_voice)


def _ms(xs):
    return dict(median_ms=1e3 * statistics.median(xs), max_ms=1e3 * max(xs), n=len(xs))


def main(argv=None):
    args = bench_parser(switches=24, steps=400, repeats=3).parse_args(argv)
    require_cuda('bench_voice_switch.py')
    from realtime_yukarin_b200 import synthetic
    from realtime_yukarin_b200.engine import Engine

    tmp = Path(tempfile.mkdtemp(prefix='bench_voice_switch_'))      # synthetic model files: never written into the tree
    eng = Engine()
    eng.set_precision('fp16')
    voices = [synthetic_voice(eng, tmp, seed) for seed in (0, 1, 2)]
    va, vb, vc = voices
    cfg = headline_config()
    n = round(T * FS)
    n_chunks = 64
    x = synthetic.synthetic_speech((n_chunks + 1) * T, stream=0)
    chunks = [np.ascontiguousarray(x[k * n:(k + 1) * n], np.float32) for k in range(n_chunks)]
    d_in = device_chunks(x, n, n_chunks)

    # ---- call: alone and as a group member ----
    sid = eng.session_create(cfg, voice=va)
    buf = np.empty(eng.session_io_geometry(sid)['max_out'])
    alone = []
    for i in range(args.switches + 2):
        eng.session_push(sid, chunks[i % n_chunks], buf)
        t0 = time.perf_counter()
        eng.session_set_voice(sid, vb if i % 2 == 0 else va)
        alone.append(time.perf_counter() - t0)
    eng.session_destroy(sid)
    members = [eng.session_create(cfg, voice=va if i % 2 == 0 else vb) for i in range(8)]
    gid = eng.group_create(members)
    bufs = [np.empty(eng.session_io_geometry(members[0])['max_out']) for _ in members]
    grouped = []
    for i in range(args.switches + 2):
        eng.group_collect(gid, eng.group_submit(gid, [chunks[(i + j) % n_chunks] for j in range(8)]), bufs)
        t0 = time.perf_counter()
        eng.session_set_voice(members[0], vc if i % 2 == 0 else va)
        grouped.append(time.perf_counter() - t0)
    eng.group_destroy(gid)
    for s in members:
        eng.session_destroy(s)
    alone, grouped = alone[2:], grouped[2:]                       # the first two calls build plans at sizes met for the first time

    # ---- stream: switching every 10 steps vs never ----
    sids = {'never': eng.session_create(cfg, voice=va), 'every_10': eng.session_create(cfg, voice=va)}
    cap = eng.session_io_geometry(sids['never'])['max_out']
    d_out, d_n = output_ring(cap)
    step_no = {v: 0 for v in sids}

    def leg(v, steps):
        eng.synchronize()
        launches0 = eng.launch_count
        t0 = time.perf_counter()
        for _ in range(steps):
            k = step_no[v]
            if v == 'every_10' and k % 10 == 0 and k:
                eng.session_set_voice(sids[v], vb if (k // 10) % 2 else va)
            eng.session_push_device(sids[v], d_in[k % n_chunks].data_ptr(), n, d_out[k % RING, 0].data_ptr(), cap,
                                    d_n[k % RING, 0].data_ptr())
            step_no[v] = k + 1
        eng.synchronize()
        return steps / (time.perf_counter() - t0), (eng.launch_count - launches0) / steps
    res = alternate(list(sids), leg, args.steps, 40, args.repeats)
    for s in sids.values():
        eng.session_destroy(s)

    # ---- latency around a switch ----
    sid = eng.session_create(cfg, voice=va)
    for k in range(20):
        eng.session_push(sid, chunks[k % n_chunks], buf)
    after = {i: [] for i in range(20)}
    for j in range(args.switches):
        eng.session_set_voice(sid, vb if j % 2 == 0 else va)
        for i in range(20):
            t0 = time.perf_counter()
            eng.session_push(sid, chunks[(j * 20 + i) % n_chunks], buf)
            after[i].append(time.perf_counter() - t0)
    eng.session_destroy(sid)
    for v in voices:
        eng.voice_destroy(v)
    shutil.rmtree(tmp, ignore_errors=True)
    steady = [t for i in range(5, 20) for t in after[i]]
    rates = {v: [r for r, _ in res[v]] for v in sids}
    line = dict(card=card(), buffer_time=T, extras=EXTRA, switches=args.switches, steps=args.steps, repeats=args.repeats,
                call=dict(alone=_ms(alone), group_member_of_8=_ms(grouped)),
                stream={v: dict(steps_per_s=statistics.median(rates[v]), steps_per_s_all=rates[v], kernels_per_step=res[v][-1][1])
                        for v in sids},
                latency=dict(**{f'step_{i}_after': _ms(after[i]) for i in range(3)}, steady=_ms(steady)))
    emit(args.out, 'bench_voice_switch', line)


if __name__ == '__main__':
    main()
