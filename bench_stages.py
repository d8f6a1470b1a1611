"""Where a streaming session's step goes: per-kernel device time of the gate, WORLD-analysis and stage-1 graphs, and the stage timeline.

One session of the headline workload (0.3 s chunks at 24 kHz, extras 0 / 0.5 / 0, base-64 seeded U-Nets, FP16, device-resident steps)
is run three ways:
  * isolated  -- one step with nothing else queued, a device synchronise before and after (--isolated steps, averaged);
  * pipelined -- --steps back-to-back steps after --warmup, as bench.py runs them; figures are per step (total over the steps / steps);
  * timeline  -- RYK_STAGE_TIMES=1: begin / end of the five stages of the last 8 pipelined steps (ryk_session_stage_times).
Kernel times come from torch.profiler with CUDA activities (CUPTI), which sees the kernels inside the session's CUDA graphs.  A kernel
is attributed to the stage whose stream it ran on; a stream's stage is named by the kernels it carries (the analysis graph's own
branch streams carry only analysis kernels).  The stage-2 kernels are further attributed to the U-Net's 16 layers by their order on
their stream: the first layer's kernel opens a forward, each k_conv_tc is the next layer (a split-K reduce belongs to the conv before
it) and the Cout = 1 kernel is the last layer.  The card's name, power limit and SM clocks are read in the same run.

    python bench_stages.py --out DIR [--steps 40 --warmup 10 --isolated 8 --f0 dio|harvest]

Writes DIR/bench_stages.json, DIR/bench_stages.md and the profiler traces, and prints the markdown.  Needs a CUDA device.  RYK_LIB
selects another build of the library (engine.py), so two builds can be profiled by the same script."""
import json
import os
import re
import tempfile
from collections import defaultdict
from pathlib import Path

os.environ['RYK_STAGE_TIMES'] = '1'             # read by ryk_session_create
os.environ.setdefault('CUDA_DEVICE_MAX_CONNECTIONS', '32')

import numpy as np  # noqa: E402

from benchlib import (FS, T, bench_parser, card, device_chunks, device_pusher, headline_config, kernel_events,  # noqa: E402
                      require_cuda, stopwatch_ms, synthetic_builtin)

CARD_FIELDS = 'name,power.limit,clocks.max.sm,clocks.sm'      # the SM clock too, read before and after the run
STAGES = ['gate_slides', 'world_analysis', 'stage1', 'stage2', 'synthesis']
# a stream's stage = the first of these whose kernel-name pattern occurs on it
STREAM_ROLES = [
    ('world_analysis', re.compile(r'k_dio|k_stonemask|k_cheaptrick|k_d4c|k_f0_out|k_hv_|crepe', re.I)),
    ('stage2', re.compile(r'k_conv_tc|splitk|k_sr_', re.I)),
    ('stage1', re.compile(r'k_set_bucket|k_s1_|stage1', re.I)),
    ('synthesis', re.compile(r'k_scrub|synth', re.I)),
    ('gate_slides', re.compile(r'k_slide<|resample|k_frame_mse|k_gate\b', re.I)),
]
REPORTED = ('gate_slides', 'world_analysis', 'stage1')


def short_name(name):
    n = name.split('(')[0] if '(' in name else name
    n = re.sub(r'^void\s+', '', n).replace('ryk::', '').replace('(anonymous namespace)::', '')
    return n.strip()


def kernels_of(prof, trace_path):
    """[(stream, name, ts_us, dur_us)] of the CUDA kernels of a torch.profiler window, through the chrome trace written to trace_path."""
    return [(e.get('args', {}).get('stream', e.get('tid')), short_name(e['name']), float(e['ts']), float(e['dur']))
            for e in kernel_events(prof, trace_path)]


def stream_roles(kernels):
    names = defaultdict(set)
    for st, n, _, _ in kernels:
        names[st].add(n)
    roles = {}
    for st, ns in names.items():
        roles[st] = next((role for role, pat in STREAM_ROLES if any(pat.search(n) for n in ns)), 'other')
    return roles


def per_kernel(kernels, n_steps):
    """{stage: {kernel: [calls per step, us per call, us per step]}} and {stage: us per step}"""
    roles = stream_roles(kernels)
    acc = defaultdict(lambda: defaultdict(lambda: [0, 0.0]))
    for st, n, _, d in kernels:
        a = acc[roles[st]][n]
        a[0] += 1
        a[1] += d
    table, totals = {}, {}
    for role, ks in acc.items():
        table[role] = {n: [c / n_steps, s / c, s / n_steps] for n, (c, s) in sorted(ks.items(), key=lambda kv: -kv[1][1])}
        totals[role] = sum(s for _, s in ks.values()) / n_steps
    return table, totals


LAYERS = [f'e{i}' for i in range(8)] + [f'd{i}' for i in range(8)]


def per_layer(kernels, n_steps):
    """{layer: [kernels per step, us per step]} of the stage-2 U-Net"""
    roles = stream_roles(kernels)
    acc = defaultdict(lambda: [0, 0.0])
    layer = {}
    for st, n, _, d in sorted((k for k in kernels if roles[k[0]] == 'stage2'), key=lambda k: (k[0], k[2])):
        if n.startswith('k_conv3x3_cin1'):
            layer[st] = 0
        elif n.startswith('k_conv_tc'):
            layer[st] = layer.get(st, -1) + 1
        elif n.startswith('k_conv3x3_cout1'):
            layer[st] = 15
        elif 'splitk' not in n:
            continue
        a = acc[LAYERS[layer[st]]]
        a[0] += 1
        a[1] += d
    return {k: [acc[k][0] / n_steps, acc[k][1] / n_steps] for k in LAYERS if k in acc}


def spans(kernels):
    """{stage: first kernel start to last kernel end (us)} of one isolated step"""
    roles = stream_roles(kernels)
    lo, hi = {}, {}
    for st, _, ts, d in kernels:
        r = roles[st]
        lo[r] = min(lo.get(r, ts), ts)
        hi[r] = max(hi.get(r, ts + d), ts + d)
    return {r: hi[r] - lo[r] for r in lo}


def main():
    ap = bench_parser(required_out=True, steps=40, warmup=10, isolated=8)
    ap.add_argument('--f0', default='dio', choices=['dio', 'harvest'])
    args = ap.parse_args()
    require_cuda('bench_stages.py')
    import torch
    from torch.profiler import ProfilerActivity, profile
    from realtime_yukarin_b200 import synthetic
    from realtime_yukarin_b200.engine import Engine

    args.out.mkdir(parents=True, exist_ok=True)
    tmp = Path(tempfile.mkdtemp(prefix='bench_stages_'))       # synthetic model files: never written into the tree
    eng = Engine()
    synthetic_builtin(eng, tmp)
    eng.set_precision('fp16')
    eng.set_f0_method(args.f0)
    cfg = headline_config()
    n = round(T * FS)
    total = args.warmup + max(args.steps, args.isolated)
    d_in = device_chunks(synthetic.synthetic_speech((total + 1) * T, stream=0), n, total)
    out_cap = (n // 1024 + 5) * 1024 + 8192
    card_before = card(CARD_FIELDS)

    def fresh_session():
        """a new session after --warmup steps, and the call that queues its next step"""
        sid = eng.session_create(cfg)
        push = device_pusher(eng, d_in, out_cap)
        for _ in range(args.warmup):
            push(sid)
        eng.synchronize()
        torch.cuda.synchronize()
        return sid, lambda: push(sid)

    acts = [ProfilerActivity.CPU, ProfilerActivity.CUDA]
    # ---- isolated steps ----
    sid, step = fresh_session()
    iso_kernels, iso_spans = [], defaultdict(list)
    for i in range(args.isolated):
        with profile(activities=acts) as prof:
            step()
            eng.synchronize()
            torch.cuda.synchronize()
        ks = kernels_of(prof, args.out / f'trace_isolated_{i}.json')
        iso_kernels += ks
        for r, v in spans(ks).items():
            iso_spans[r].append(v)
    eng.session_destroy(sid)
    iso_table, iso_totals = per_kernel(iso_kernels, args.isolated)
    iso_layers = per_layer(iso_kernels, args.isolated)

    # ---- pipelined steps ----
    sid, step = fresh_session()
    with profile(activities=acts) as prof:
        for _ in range(args.steps):
            step()
        eng.synchronize()
        torch.cuda.synchronize()
    pipe_kernels = kernels_of(prof, args.out / 'trace_pipelined.json')
    pipe_table, pipe_totals = per_kernel(pipe_kernels, args.steps)
    pipe_layers = per_layer(pipe_kernels, args.steps)
    eng.session_destroy(sid)

    # ---- stage timeline, profiler off ----
    sid, step = fresh_session()
    ms = stopwatch_ms(eng, step, 0, args.steps)
    st, en = eng.session_stage_times(sid)
    eng.session_destroy(sid)
    # gate of step k against the end of stage 1 of step k-2 (> 0: the gate started after it)
    gate_vs_s1 = [float(st[i, 0] - en[i - 2, 2]) for i in range(2, len(st))]

    res = dict(card=card_before, card_after=card(CARD_FIELDS), f0=args.f0, steps=args.steps, warmup=args.warmup, isolated=args.isolated,
               lib=os.environ.get('RYK_LIB', 'realtime_yukarin_b200/csrc/libryk.so'),
               isolated_us=iso_table, isolated_stage_us=iso_totals,
               isolated_stage_span_us={r: float(np.mean(v)) for r, v in iso_spans.items()},
               pipelined_us=pipe_table, pipelined_stage_us=pipe_totals,
               stage2_layers=dict(isolated_us=iso_layers, pipelined_us=pipe_layers),
               timeline=dict(stages=STAGES, start_ms=np.round(st, 4).tolist(), end_ms=np.round(en, 4).tolist(),
                             ms_per_step=ms / args.steps, gate_start_minus_stage1_end_of_k_minus_2_ms=np.round(gate_vs_s1, 4).tolist()))
    (args.out / 'bench_stages.json').write_text(json.dumps(res, indent=1))

    lines = [f'card: {res["card"]} (after: {res["card_after"]}); f0 {args.f0}; library {res["lib"]}', '']
    for role in REPORTED:
        lines += [f'### {role}: {iso_totals.get(role, 0):.1f} us of kernels per isolated step (span '
                  f'{res["isolated_stage_span_us"].get(role, 0):.1f} us), {pipe_totals.get(role, 0):.1f} us per pipelined step', '',
                  '| kernel | calls / step | isolated us / call | isolated us / step | pipelined us / step |', '|---|---|---|---|---|']
        names = list(iso_table.get(role, {})) + [k for k in pipe_table.get(role, {}) if k not in iso_table.get(role, {})]
        for k in names:
            c, per, tot = iso_table.get(role, {}).get(k, [0, 0, 0])
            pt = pipe_table.get(role, {}).get(k, [0, 0, 0])[2]
            lines.append(f'| `{k}` | {c:g} | {per:.2f} | {tot:.2f} | {pt:.2f} |')
        lines.append('')
    lines += [f'### stage 2 per layer: {sum(v[1] for v in iso_layers.values()):.1f} us of kernels per isolated step, '
              f'{sum(v[1] for v in pipe_layers.values()):.1f} us per pipelined step', '',
              '| layer | kernels / step | isolated us / step | pipelined us / step |', '|---|---|---|---|']
    for k in LAYERS:
        c, iso = iso_layers.get(k, [0, 0])
        lines.append(f'| {k} | {c:g} | {iso:.2f} | {pipe_layers.get(k, [0, 0])[1]:.2f} |')
    lines.append('')
    other = {r: v for r, v in pipe_totals.items() if r not in REPORTED}
    lines += ['other stages, pipelined us of kernels per step: ' + ', '.join(f'{r} {v:.1f}' for r, v in sorted(other.items())), '',
              f'timeline (RYK_STAGE_TIMES=1, profiler off): {res["timeline"]["ms_per_step"]:.4f} ms per step over {args.steps} steps', '',
              '| step | ' + ' | '.join(STAGES) + ' |', '|---' * (len(STAGES) + 1) + '|']
    for i in range(len(st)):
        lines.append(f'| {i} | ' + ' | '.join(f'{st[i, a]:.3f}-{en[i, a]:.3f}' for a in range(len(STAGES))) + ' |')
    lines += ['', 'gate start of step k minus stage-1 end of step k-2 (ms): ' + ', '.join(f'{v:.3f}' for v in gate_vs_s1)]
    md = '\n'.join(lines) + '\n'
    (args.out / 'bench_stages.md').write_text(md)
    print(md)


if __name__ == '__main__':
    main()
