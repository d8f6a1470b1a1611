"""Cost of changing a running group's members between steps (ryk_group_add / ryk_group_remove).

Three measurements on one engine, precision 1, 0.3 s chunks, extras 0 / 0.5 / 0, one full-width synthetic voice (seed 0):
  * change calls: a running group of B members (B = 1..8) takes a running session in (group_add, B -> B + 1) and lets it go again
    (group_remove, B + 1 -> B).  Host wall time of each call (it returns with the device synchronised and the new plan built), median
    over --repeats.
  * first step after a change: host time of the group_push_device call right after the change, which captures the group's forward and
    the members' stage-2 prologue / epilogue graphs anew, against the host time of a step with captured graphs (both medians; the
    device is idle when each call starts).
  * churn: device-resident chunks/s of a 4-member group where the last member leaves and rejoins every 10 steps (two change calls, its
    stream state carried over), against the same group with fixed membership.  Legs alternate over --rounds rounds; each leg runs
    --steps steps after --warmup, timed on the host clock from an idle device to an idle device.  Reported: median chunks/s.
The card's name and power limit are recorded with the numbers.

    python bench_group_churn.py [--out DIR] [--repeats 7 --steps 100 --warmup 10 --rounds 3]

Prints one JSON line (and writes it to DIR/bench_group_churn.json with --out).  Needs a CUDA device; there is no CPU path."""
import shutil
import statistics
import tempfile
import time
from pathlib import Path

from benchlib import EXTRA, FS, T, bench_parser, card, device_chunks, emit, headline_config, require_cuda, synthetic_voice

BS = list(range(1, 9))


def main():
    args = bench_parser(repeats=7, steps=100, warmup=10, rounds=3).parse_args()
    require_cuda('bench_group_churn.py')
    import torch
    from realtime_yukarin_b200 import synthetic
    from realtime_yukarin_b200.engine import Engine

    tmp = Path(tempfile.mkdtemp(prefix='bench_group_churn_'))       # synthetic model files: never written into the tree
    eng = Engine()
    eng.set_precision('fp16')
    voice = synthetic_voice(eng, tmp)
    cfg = headline_config()
    n = round(T * FS)
    n_chunks = 64
    d_in = device_chunks(synthetic.synthetic_speech((n_chunks + 1) * T, stream=0), n, n_chunks)
    sids = [eng.session_create(cfg, voice=voice) for _ in range(max(BS) + 1)]
    cap = eng.session_io_geometry(sids[0])['max_out']
    d_out = torch.empty((len(sids), cap), dtype=torch.float64, device='cuda')
    d_n = torch.zeros((len(sids), 1), dtype=torch.int32, device='cuda')
    step_no = {s: 0 for s in sids}

    def push_group(gid):
        members = eng.group_members(gid)
        eng.group_push_device(gid, [d_in[step_no[s] % n_chunks].data_ptr() for s in members], n, [d_out[s - sids[0]].data_ptr() for s in members],
                              cap, [d_n[s - sids[0]].data_ptr() for s in members])
        for s in members:
            step_no[s] += 1

    def push_alone(s):
        eng.session_push_device(s, d_in[step_no[s] % n_chunks].data_ptr(), n, d_out[s - sids[0]].data_ptr(), cap, d_n[s - sids[0]].data_ptr())
        step_no[s] += 1

    def host_ms(call):
        t0 = time.perf_counter()
        call()
        return (time.perf_counter() - t0) * 1e3

    def idle_step_ms(gid):
        eng.synchronize()
        return host_ms(lambda: push_group(gid))

    # ---- change calls and the first step after each, at B = 1..8 ----
    changes = []
    joiner = sids[-1]
    for _ in range(2):
        push_alone(joiner)                        # the joiner is a running session with its own stage-2 plans
    for B in BS:
        gid = eng.group_create(sids[:B])
        for _ in range(3):
            push_group(gid)
        add, rem, first_add, first_rem, steady = [], [], [], [], []
        for _ in range(args.repeats):
            eng.synchronize()
            add.append(host_ms(lambda: eng.group_add(gid, joiner)))
            first_add.append(idle_step_ms(gid))
            steady.append(idle_step_ms(gid))
            eng.synchronize()
            rem.append(host_ms(lambda: eng.group_remove(gid, joiner)))
            first_rem.append(idle_step_ms(gid))
            steady.append(idle_step_ms(gid))
            push_alone(joiner)
        eng.synchronize()
        eng.group_destroy(gid)
        changes.append(dict(B=B, add_ms=statistics.median(add), remove_ms=statistics.median(rem),
                            first_step_after_add_ms=statistics.median(first_add), first_step_after_remove_ms=statistics.median(first_rem),
                            steady_step_ms=statistics.median(steady), add_ms_all=add, remove_ms_all=rem))

    # ---- churn: 4 members, the last one leaves and rejoins every 10 steps, against fixed membership ----
    members = sids[:4]

    def leg(churn):
        gid = eng.group_create(members)
        for _ in range(args.warmup):
            push_group(gid)
        eng.synchronize()
        t0 = time.perf_counter()
        for k in range(args.steps):
            if churn and k % 10 == 9:
                eng.group_remove(gid, members[-1])
                eng.group_add(gid, members[-1])
            push_group(gid)
        eng.synchronize()
        s = time.perf_counter() - t0
        eng.group_destroy(gid)
        return len(members) * args.steps / s

    leg(True)                                     # first-use costs outside the rounds
    rates = {'fixed': [], 'churn': []}
    for _ in range(args.rounds):
        rates['fixed'].append(leg(False))
        rates['churn'].append(leg(True))
    for s in sids:
        eng.session_destroy(s)
    eng.voice_destroy(voice)
    shutil.rmtree(tmp, ignore_errors=True)
    churn = dict(members=len(members), change_every=10, steps=args.steps, warmup=args.warmup, rounds=args.rounds,
                 fixed_chunks_per_s=statistics.median(rates['fixed']), churn_chunks_per_s=statistics.median(rates['churn']),
                 fixed_all=rates['fixed'], churn_all=rates['churn'])
    line = dict(card=card(), buffer_time=T, extras=EXTRA, repeats=args.repeats, changes=changes, churn=churn)
    emit(args.out, 'bench_group_churn', line)


if __name__ == '__main__':
    main()
