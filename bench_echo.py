"""Cost of the echo canceller on the headline stream (precision 1, 0.3 s chunks at 24 kHz, extras 0 / 0.5 / 0, full-width synthetic
voice), with the canceller off and at 16, 32 and 64 taps:

  alone  one session: steps/s of ryk_session_push_device in blocks of --block (the device drains between blocks, as in bench.py's
         sustained figure), and the submit-to-collect latency of blocking host-API steps (ryk_session_echo_reference, then
         ryk_session_submit and ryk_session_collect), median and 95th percentile
  group  8 sessions in one group: steps/s and latency of blocking ryk_group_submit / ryk_group_collect steps, every member handed a
         far end first

Every variant's far end is a second speech stream, so the filters adapt on every frame.  The variants alternate within each of --repeats
rounds after --warmup steps each.  After the timed rounds one torch.profiler window over --profile_steps steps of each lone session
gives k_aec_scan's kernel time per step (and the gate stage's kernels for comparison).  The card's name and power limit are recorded
with the numbers.

    python bench_echo.py [--out DIR] [--steps 1000 --block 100 --latency_steps 200 --group_steps 300 --warmup 30 --repeats 3]

Prints one JSON line (and writes it to DIR/bench_echo.json with --out).  Needs a CUDA device; there is no CPU path."""
import shutil
import statistics
import tempfile
import time
from pathlib import Path

import numpy as np

from benchlib import (EXTRA, FS, RING, T, bench_parser, card, device_chunks, emit, headline_config, kernel_durations, output_ring,
                      require_cuda, synthetic_voice, throughput)

VARIANTS = ('off', 16, 32, 64)
GROUP = 8


def main(argv=None):
    args = bench_parser(steps=1000, block=100, latency_steps=200, group_steps=300, warmup=30, repeats=3,
                        profile_steps=20).parse_args(argv)
    require_cuda('bench_echo.py')
    from realtime_yukarin_b200 import synthetic
    from realtime_yukarin_b200.engine import Engine

    tmp = Path(tempfile.mkdtemp(prefix='bench_echo_'))              # synthetic model files: never written into the tree
    eng = Engine()
    eng.set_precision('fp16')
    voice = synthetic_voice(eng, tmp)
    cfg = headline_config()
    n = round(T * FS)
    n_chunks = 64
    x = synthetic.synthetic_speech((n_chunks + 1) * T, stream=0)
    far = (0.5 * synthetic.synthetic_speech((n_chunks + 1) * T, stream=1)).astype(np.float32)
    mic_chunks = [np.ascontiguousarray(x[k * n:(k + 1) * n]) for k in range(n_chunks)]
    far_chunks = [np.ascontiguousarray(far[k * n:(k + 1) * n]) for k in range(n_chunks)]
    d_in = device_chunks(x, n, n_chunks)

    def make(v):
        sid = eng.session_create(cfg, voice=voice)
        if v != 'off':
            eng.session_echo_cancel(sid, taps=v)
        return sid
    alone = {v: make(v) for v in VARIANTS}
    groups = {}
    for v in VARIANTS:
        members = [make(v) for _ in range(GROUP)]
        groups[v] = (eng.group_create(members), members)
    cap = eng.session_io_geometry(alone['off'])['max_out']
    d_out, d_n = output_ring(cap)
    buf = np.empty(cap)
    gbufs = [np.empty(cap) for _ in range(GROUP)]
    step_no = {v: 0 for v in VARIANTS}
    gstep_no = {v: 0 for v in VARIANTS}

    def push_device(v):
        k = step_no[v]
        if v != 'off':
            eng.session_echo_reference(alone[v], far_chunks[k % n_chunks])
        eng.session_push_device(alone[v], d_in[k % n_chunks].data_ptr(), n, d_out[k % RING, 0].data_ptr(), cap, d_n[k % RING, 0].data_ptr())
        step_no[v] = k + 1

    def push_host(v):
        k = step_no[v]
        t0 = time.perf_counter()
        if v != 'off':
            eng.session_echo_reference(alone[v], far_chunks[k % n_chunks])
        eng.session_collect(alone[v], eng.session_submit(alone[v], mic_chunks[k % n_chunks]), buf)
        step_no[v] = k + 1
        return time.perf_counter() - t0

    def push_group(v):
        gid, members = groups[v]
        k = gstep_no[v]
        t0 = time.perf_counter()
        if v != 'off':
            for j, sid in enumerate(members):
                eng.session_echo_reference(sid, far_chunks[(k + j) % n_chunks])
        eng.group_collect(gid, eng.group_submit(gid, [mic_chunks[(k + j) % n_chunks] for j in range(GROUP)]), gbufs)
        gstep_no[v] = k + 1
        return time.perf_counter() - t0

    def leg_latency(fn, v, steps):
        eng.synchronize()
        t0 = time.perf_counter()
        lat = [fn(v) for _ in range(steps)]
        return steps / (time.perf_counter() - t0), lat

    for v in VARIANTS:
        throughput(eng, lambda: push_device(v), args.warmup, args.block)
        leg_latency(push_host, v, args.warmup)
        leg_latency(push_group, v, args.warmup)
    res = {v: dict(alone_steps_per_s=[], alone_latency_ms=[], group_steps_per_s=[], group_latency_ms=[]) for v in VARIANTS}
    for _ in range(args.repeats):
        for v in VARIANTS:
            r = res[v]
            r['alone_steps_per_s'].append(throughput(eng, lambda: push_device(v), args.steps, args.block))
            r['alone_latency_ms'].extend(1e3 * t for t in leg_latency(push_host, v, args.latency_steps)[1])
            rate, lat = leg_latency(push_group, v, args.group_steps)
            r['group_steps_per_s'].append(rate)
            r['group_latency_ms'].extend(1e3 * t for t in lat)

    # kernel times: one profiler window over the lone sessions, one variant after the other
    def profiled_steps():
        for v in VARIANTS:
            for _ in range(args.profile_steps):
                push_host(v)
    durations = kernel_durations(eng, tmp, profiled_steps, ('k_aec_scan', 'k_dn_forward', 'k_dn_inverse'))
    scans, fwd, inv = durations['k_aec_scan'], durations['k_dn_forward'], durations['k_dn_inverse']
    tapped = [v for v in VARIANTS if v != 'off']
    kernels = {}
    for i, v in enumerate(tapped):
        s = scans[i * args.profile_steps:(i + 1) * args.profile_steps]
        kernels[str(v)] = dict(k_aec_scan_us_median=statistics.median(s), k_aec_scan_us_max=max(s))
    kernels['k_dn_forward_us_median'] = statistics.median(fwd) if fwd else None
    kernels['k_dn_inverse_us_median'] = statistics.median(inv) if inv else None

    for gid, _ in groups.values():
        eng.group_destroy(gid)
    for sid in list(alone.values()) + [s for _, members in groups.values() for s in members]:
        eng.session_destroy(sid)
    eng.voice_destroy(voice)
    shutil.rmtree(tmp, ignore_errors=True)

    def summary(r):
        lat, glat = sorted(r['alone_latency_ms']), sorted(r['group_latency_ms'])
        return dict(alone_steps_per_s=statistics.median(r['alone_steps_per_s']), alone_steps_per_s_all=r['alone_steps_per_s'],
                    alone_latency_ms_median=statistics.median(lat), alone_latency_ms_p95=lat[int(0.95 * (len(lat) - 1))],
                    group_steps_per_s=statistics.median(r['group_steps_per_s']), group_steps_per_s_all=r['group_steps_per_s'],
                    group_latency_ms_median=statistics.median(glat), group_latency_ms_p95=glat[int(0.95 * (len(glat) - 1))])
    line = dict(card=card(), buffer_time=T, extras=EXTRA, group=GROUP, steps=args.steps, block=args.block,
                latency_steps=args.latency_steps, group_steps=args.group_steps, warmup=args.warmup, repeats=args.repeats,
                variants={str(v): summary(res[v]) for v in VARIANTS}, kernels=kernels)
    emit(args.out, 'bench_echo', line)


if __name__ == '__main__':
    main()
