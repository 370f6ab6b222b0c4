"""Timeline of the configs[1] training step as bench.py replays it (GUM, T = 1, B = 256, h = 512, 3xTF32, one CUDA graph per
resident batch, L2 flushed before each replay).

Prints, and writes as JSON under --out:
  * the card, its power limit and its SM clock (nvidia-smi, read in the same run);
  * the graph-replay step time over --replays replays: median, spread, percentiles;
  * the captured graph's nodes and edges (cudaGraphGetEdges_v2): the edge type says which dependencies are programmatic;
  * one replay from torch.profiler (CUDA activity): start and end of every kernel and memset with its stream, and for each
    node of the main stream the gap from the end of its main-stream predecessor to its own start, next to the last end so
    far on each side stream (a join is late when that end is after the main-stream predecessor's).

Which stream a node was enqueued on is taken from one profiled eager step (the replay runs the graph's branches on streams
of its own); nodes of the replay are matched to the eager launches by kernel name, grid and block, in order.

usage: python scripts/t1_chain_timeline.py [--out DIR] [--replays N] [--precision P]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

LSTM_DIM, BATCH = 512, 256   # bench.py configs[1]


def card():
    q = 'name,power.limit,clocks.sm,clocks.max.sm'
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=' + q, '--format=csv,noheader', '-i', '0'], capture_output=True,
                             text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as exc:
        out = 'nvidia-smi unavailable: {}'.format(exc)
    return {'query': q, 'value': out}


def bench_step(precision):
    """The objects and the step of bench.py (single GPU, device-resident).  This restates bench.py by hand: the network,
    optimiser and seeds of `main()` (rng 1234, `gum_network(..., seed=0)`, Adam at 1e-3, four resident batches), its
    `hyper` / `adam_state` tensors and `device_step()` (bench.py:283-344 at the time of writing); keep them in step with
    bench.py when it changes."""
    from pyprob_b200 import synthetic
    from pyprob_b200._lib import call, ptr
    from pyprob_b200.network import BatchStruct
    from pyprob_b200.util import Optimizer
    dev = torch.device('cuda:0')
    torch.cuda.set_device(dev)
    rng = np.random.default_rng(1234)
    net = synthetic.gum_network(lstm_dim=LSTM_DIM, precision=precision, seed=0)
    net._optimizer_type, net._learning_rate_init, net._weight_decay = Optimizer.ADAM, 1e-3, 0.0
    net._create_optimizer()
    net._sync_native()
    nparams = net._arena.numel()
    grad = torch.zeros(nparams, device=dev)
    net._arena.grad = grad
    encs = [synthetic.gum_batch(rng, BATCH).encode(net) for _ in range(4)]
    hyper = torch.tensor([1e-3, 0.9, 0.999, 1e-8, 0.0, 1.0], dtype=torch.float32, device=dev)
    adam_state = torch.zeros(4, dtype=torch.int32, device=dev)
    loss = torch.empty((), device=dev)
    status = torch.zeros(1, dtype=torch.int32, device=dev)
    hosts = [torch.from_numpy(enc.pack().copy()).pin_memory() for enc in encs]
    resident = [h.to(dev) for h in hosts]
    cur = torch.empty_like(resident[0])
    bs = BatchStruct()
    call('ppb_batch_from_image', hosts[0].data_ptr(), cur.data_ptr(), hosts[0].numel(), C.byref(bs))
    need = net._ensure_workspace(encs[0])

    def device_step(i):
        st = torch.cuda.current_stream().cuda_stream
        cur.copy_(resident[i % 4], non_blocking=True)
        grad.zero_()
        call('ppb_ic_loss_forward', net._handle, ptr(net._arena.data), C.byref(bs), ptr(net._workspace), need, precision,
             ptr(loss), ptr(status), None, 1, st)
        call('ppb_ic_loss_backward', net._handle, ptr(net._arena.data), ptr(grad), C.byref(bs), ptr(net._workspace), need,
             precision, 1.0, st)
        call('ppb_adam_step_dev', ptr(net._arena.data), ptr(grad), ptr(net._exp_avg), ptr(net._exp_avg_sq), nparams,
             ptr(hyper), ptr(adam_state), st)
    return dev, device_step, status


def capture(device_step, i, keep_graph=False):
    g = torch.cuda.CUDAGraph(keep_graph=keep_graph)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        with torch.cuda.graph(g, stream=side):
            device_step(i)
    torch.cuda.current_stream().wait_stream(side)
    return g


# ---- graph edges through the CUDA runtime torch has loaded -------------------------------------------------------------
def _cudart():
    with open('/proc/self/maps') as f:
        paths = sorted({ln.split()[-1] for ln in f if 'libcudart.so' in ln})
    if not paths:
        raise RuntimeError('libcudart is not loaded in this process')
    return C.CDLL(paths[0])


def _demangle(name):
    try:
        cxx = C.CDLL('libstdc++.so.6')
        cxx.__cxa_demangle.restype = C.c_void_p
        st = C.c_int()
        p = cxx.__cxa_demangle(name.encode(), None, None, C.byref(st))
        if st.value == 0 and p:
            s = C.string_at(p).decode()
            C.CDLL(None).free(C.c_void_p(p))
            return s
    except OSError:
        pass
    return name


class _KParams(C.Structure):   # cudaKernelNodeParams
    _fields_ = [('func', C.c_void_p), ('grid', C.c_uint * 3), ('block', C.c_uint * 3), ('smem', C.c_uint),
                ('params', C.c_void_p), ('extra', C.c_void_p)]


class _EdgeData(C.Structure):  # cudaGraphEdgeData
    _fields_ = [('from_port', C.c_ubyte), ('to_port', C.c_ubyte), ('type', C.c_ubyte), ('reserved', C.c_ubyte * 5)]


NODE_TYPES = {0: 'kernel', 1: 'memcpy', 2: 'memset', 3: 'host', 4: 'graph', 5: 'empty', 6: 'wait_event',
              7: 'event_record', 8: 'ext_sem_signal', 9: 'ext_sem_wait', 10: 'mem_alloc', 11: 'mem_free',
              12: 'batch_mem_op', 13: 'conditional'}
EDGE_TYPES = {0: 'full', 1: 'programmatic'}


def graph_dump(graph):
    rt = _cudart()
    g = C.c_void_p(graph)
    n = C.c_size_t(0)
    if rt.cudaGraphGetNodes(g, None, C.byref(n)):
        raise RuntimeError('cudaGraphGetNodes failed')
    nodes = (C.c_void_p * n.value)()
    rt.cudaGraphGetNodes(g, nodes, C.byref(n))
    index = {nodes[i]: i for i in range(n.value)}
    out_nodes = []
    for i in range(n.value):
        t = C.c_int()
        rt.cudaGraphNodeGetType(C.c_void_p(nodes[i]), C.byref(t))
        d = {'id': i, 'type': NODE_TYPES.get(t.value, str(t.value))}
        if t.value == 0:
            kp = _KParams()
            if rt.cudaGraphKernelNodeGetParams(C.c_void_p(nodes[i]), C.byref(kp)) == 0:
                nm = C.c_char_p()
                name = '?'
                if rt.cudaFuncGetName(C.byref(nm), C.c_void_p(kp.func)) == 0 and nm.value:
                    name = _demangle(nm.value.decode())
                d.update(name=short(name), grid=list(kp.grid), block=list(kp.block), smem=kp.smem)
        out_nodes.append(d)
    ne = C.c_size_t(0)
    if rt.cudaGraphGetEdges_v2(g, None, None, None, C.byref(ne)):
        raise RuntimeError('cudaGraphGetEdges_v2 failed')
    fr, to = (C.c_void_p * ne.value)(), (C.c_void_p * ne.value)()
    ed = (_EdgeData * ne.value)()
    rt.cudaGraphGetEdges_v2(g, fr, to, ed, C.byref(ne))
    edges = [{'from': index[fr[i]], 'to': index[to[i]], 'type': EDGE_TYPES.get(ed[i].type, str(ed[i].type)),
              'from_port': ed[i].from_port} for i in range(ne.value)]
    return out_nodes, edges


def label(n):
    if n['type'] != 'kernel':
        return '#{} {}'.format(n['id'], n['type'])
    return '#{} {} grid {}'.format(n['id'], n.get('name', '?'), 'x'.join(str(v) for v in n.get('grid', [])))


def short(name):
    name = name.replace('(anonymous namespace)::', '')
    if len(name) <= 60:
        return name
    base = name.split('<')[0].split('(')[0]
    tags = [t for t in ('NllRowEpi', 'CellBwdT1Epi', 'FillFunctor') if t in name]
    return base + ('<{}>'.format(','.join(tags)) if tags else '<...>')


# ---- profiler timeline ----------------------------------------------------------------------------------------------------
def gpu_events(prof, out_dir, tag):
    path = os.path.join(out_dir, 'trace_{}.json'.format(tag))
    prof.export_chrome_trace(path)
    with open(path) as f:
        tr = json.load(f)
    os.remove(path)   # traces are large: the table below is what is kept
    evs = []
    for e in tr.get('traceEvents', []):
        if e.get('ph') != 'X' or e.get('cat') not in ('kernel', 'gpu_memset', 'gpu_memcpy'):
            continue
        a = e.get('args', {})
        evs.append({'cat': e['cat'], 'name': short(e['name']), 'ts': float(e['ts']), 'end': float(e['ts']) + float(e['dur']),
                    'stream': a.get('stream'), 'corr': a.get('correlation'), 'grid': a.get('grid'), 'block': a.get('block')})
    return evs


def key_of(e):
    return (e['cat'], e['name'], str(e['grid']), str(e['block']))


def timeline(eager, replay):
    """Roles (stream of enqueue, launch order) from the eager step; times from the replay."""
    eager = sorted(eager, key=lambda e: (e['corr'] or 0, e['ts']))
    names = {}
    for e in eager:   # streams named in order of first enqueue: main (the batch copy), then s1, s2
        if e['stream'] not in names:
            names[e['stream']] = 'main' if not names else 's{}'.format(len(names))
    for i, e in enumerate(eager):
        e['role'], e['order'] = names[e['stream']], i
    by_key = {}
    for e in eager:
        by_key.setdefault(key_of(e), []).append(e)
    rows, ambiguous = [], set()
    seen = {}
    t0 = min(e['ts'] for e in replay)
    for r in sorted(replay, key=lambda e: e['ts']):
        k = key_of(r)
        cand = by_key.get(k, [])
        j = seen.get(k, 0)
        seen[k] = j + 1
        if j >= len(cand):
            rows.append(dict(r, role='?', order=10 ** 6, start_us=r['ts'] - t0, end_us=r['end'] - t0))
            continue
        if len({c['role'] for c in cand}) > 1:
            ambiguous.add(k[1])
        rows.append(dict(r, role=cand[j]['role'], order=cand[j]['order'], start_us=r['ts'] - t0, end_us=r['end'] - t0))
    rows.sort(key=lambda r: r['start_us'])
    prev_main = None
    for r in rows:
        r['dur_us'] = r['end_us'] - r['start_us']
        if r['role'] != 'main':
            continue
        if prev_main is not None:
            r['gap_us'] = r['start_us'] - prev_main['end_us']
        for s in ('s1', 's2'):
            ends = [q['end_us'] for q in rows if q['role'] == s and q['order'] < r['order']]
            r[s + '_end_us'] = max(ends) if ends else None
        prev_main = r
    return rows, sorted(ambiguous)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None, help='directory for timeline.json (default: a new temporary directory)')
    ap.add_argument('--replays', type=int, default=300)
    ap.add_argument('--precision', type=int, default=0)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('t1_chain_timeline: no CUDA device')
    out_dir = args.out or tempfile.mkdtemp(prefix='t1_timeline_')
    os.makedirs(out_dir, exist_ok=True)
    from pyprob_b200 import _lib
    result = {'card': card()}
    dev, device_step, status = bench_step(args.precision)
    for i in range(5):
        device_step(i)
    torch.cuda.synchronize()
    l0 = _lib.call('ppb_launch_count')
    device_step(0)
    torch.cuda.synchronize()
    result['launches_per_step'] = int(_lib.call('ppb_launch_count') - l0)
    graphs = [capture(device_step, i) for i in range(4)]
    for i in range(10):
        graphs[i % 4].replay()
    torch.cuda.synchronize()
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)

    # step time: bench.py's timed loop
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.replays)]
    stream = torch.cuda.current_stream()
    for i in range(args.replays):
        flush.zero_()
        ev[i][0].record(stream)
        graphs[i % 4].replay()
        ev[i][1].record(stream)
    torch.cuda.synchronize()
    ms = np.array([a.elapsed_time(b) for a, b in ev])
    result['step_ms'] = {'n': int(ms.size), 'median': float(np.median(ms)), 'min': float(ms.min()), 'max': float(ms.max()),
                         'p10': float(np.percentile(ms, 10)), 'p90': float(np.percentile(ms, 90))}
    assert int(status.item()) == 0

    # the captured graph of batch 0
    gk = capture(device_step, 0, keep_graph=True)
    nodes, edges = graph_dump(gk.raw_cuda_graph())
    result['graph'] = {'nodes': nodes, 'edges': edges}
    del gk

    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        device_step(0)
        torch.cuda.synchronize()
    eager = gpu_events(prof, out_dir, 'eager')
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(3):
            flush.zero_()
            graphs[0].replay()
        torch.cuda.synchronize()
    evs = gpu_events(prof, out_dir, 'replay')
    # every node of one graph launch carries the correlation id of that cudaGraphLaunch: the last replay is the last group
    # with more than one event; without such groups, what follows the last L2 flush (the longest fill) is the replay
    groups = {}
    for e in evs:
        groups.setdefault(e['corr'], []).append(e)
    many = [g for g in groups.values() if len(g) > 1]
    if many:
        replay = max(many, key=lambda g: min(e['ts'] for e in g))
    else:
        fills = [e for e in evs if 'FillFunctor' in e['name'] or e['cat'] == 'gpu_memset']
        longest = max(e['end'] - e['ts'] for e in fills)
        last_flush = max((e for e in fills if e['end'] - e['ts'] > 0.5 * longest), key=lambda e: e['ts'])
        replay = [e for e in evs if e['ts'] >= last_flush['end']]
    rows, ambiguous = timeline(eager, replay)
    result['timeline'] = rows
    result['ambiguous_keys'] = ambiguous

    with open(os.path.join(out_dir, 'timeline.json'), 'w') as f:
        json.dump(result, f, indent=1)

    print('card: {} ({})'.format(result['card']['value'], result['card']['query']))
    print('launches per eager step: {}'.format(result['launches_per_step']))
    s = result['step_ms']
    print('graph replay, L2 flushed: median {:.4f} ms, min {:.4f}, p10 {:.4f}, p90 {:.4f}, max {:.4f} over {}'.format(
        s['median'], s['min'], s['p10'], s['p90'], s['max'], s['n']))
    print('\ngraph edges (from -> to, type):')
    for e in edges:
        print('  {:<60} -> {:<60} {}{}'.format(label(nodes[e['from']]), label(nodes[e['to']]), e['type'],
                                             '' if e['from_port'] == 0 else ' (port {})'.format(e['from_port'])))
    print('\none replay (µs from its first node; gap: start after the end of the previous main-stream node; s1/s2 end: '
          'last end so far of the side-stream nodes enqueued before it):')
    print('{:<5} {:>8} {:<48} {:>8} {:>8} {:>7} {:>7} {:>8} {:>8}'.format('role', 'stream', 'node', 'start', 'end', 'dur',
                                                                        'gap', 's1 end', 's2 end'))
    f = lambda v: '' if v is None else '{:.1f}'.format(v)  # noqa: E731
    for r in rows:
        print('{:<5} {:>8} {:<48} {:>8.1f} {:>8.1f} {:>7.1f} {:>7} {:>8} {:>8}'.format(
            r['role'], str(r['stream']), r['name'][:48], r['start_us'], r['end_us'], r['dur_us'], f(r.get('gap_us')),
            f(r.get('s1_end_us')), f(r.get('s2_end_us'))))
    if ambiguous:
        print('matched by order across streams (same name, grid and block on several streams): ' + ', '.join(ambiguous))
    print('\nwritten: ' + os.path.join(out_dir, 'timeline.json'))


if __name__ == '__main__':
    main()
