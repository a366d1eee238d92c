"""Marginal cost of every layer INSIDE the persistent conv-group launch (MobileNet-v2 int8 conv path, batch 32): the step is
timed with the group of all layers and then with a group of every layer but one, bound to the same tensors; the difference is
what that layer costs in situ (cache state, co-scheduling with the other layers), next to its algorithmic bytes and the HBM
time those bytes would take.  "alone" splits the step: the launches outside the group (stem, strided convs) and the group's
launches, each captured in a CUDA graph of its own and replayed back to back; group_launches_ms splits the group into its
shallow-kernel and conv-group-kernel launches (torch.profiler).  Usage (on the GPU): python tools/group_layer_costs.py > layer_costs.json"""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from mnn_b200 import mnn_file  # noqa: E402
from mnn_b200.backend import ConvGroupExecution  # noqa: E402
from mnn_b200.session import ConvPathSession  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MODEL = os.path.join(ROOT, "tests", "golden", "mbv2_int8.mnn")
PEAK_GBS = 3350.0     # H100 SXM data-sheet HBM3 bandwidth


def time_fn(stream, fn, steps=40, warm=5, reps=5):
    """median over `reps` windows of the device time per call of fn (which enqueues on `stream`)"""
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(warm):
        fn()
    out = []
    for _ in range(reps):
        with torch.cuda.stream(stream):
            ev0.record()
        for _ in range(steps):
            fn()
        with torch.cuda.stream(stream):
            ev1.record()
        stream.synchronize()
        out.append(ev0.elapsed_time(ev1) / steps)
    out.sort()
    return out[len(out) // 2]


def time_steps(sess, steps=40, warm=5, reps=5):
    return time_fn(sess.stream, sess.run, steps, warm, reps)


def time_alone(sess, enqueue, steps=200, reps=9):
    """one CUDA graph of `enqueue` alone, replayed back to back: that launch's own time per step"""
    with torch.cuda.stream(sess.stream):
        enqueue()
    sess.stream.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=sess.stream):
        enqueue()

    def replay():
        with torch.cuda.stream(sess.stream):
            g.replay()
    return time_fn(sess.stream, replay, steps, 20, reps)


def split(sess):
    """the step's own time, the singles' (stem, strided convs) alone and the group launch alone"""
    def singles():
        for node, ex, x, y in sess.singles:
            assert ex.onExecute([x], [y]) == 0, node.name

    def group():
        assert sess.group.onExecute() == 0

    return {"step_ms": time_alone(sess, lambda: (singles(), group())), "singles_ms": time_alone(sess, singles),
            "group_ms": time_alone(sess, group), "group_launches_ms": per_launch(sess, group)}


def per_launch(sess, enqueue, steps=50):
    """the group's launches (the shallow kernel, then the conv-group kernel) timed one by one under torch.profiler: mean device
    ms per step of each kernel"""
    from torch.profiler import ProfilerActivity, profile
    for _ in range(5):
        enqueue()
    sess.stream.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            enqueue()
        sess.stream.synchronize()
    out = {}
    for ev in prof.key_averages():
        for name in ("conv_group_shallow_wgmma_kernel", "conv_group_wgmma_kernel"):
            if name in ev.key:
                out[name] = round(ev.device_time_total / 1e3 / steps, 4)
    return out


def main():
    sess = ConvPathSession(mnn_file.load(open(MODEL, "rb").read()), 32)
    members = [l for l in sess.layers if ConvGroupExecution.groupable(l[1])]

    def rebuild(skip):
        keep = [l for i, l in enumerate(members) if i != skip]
        sess.graph = None
        sess.group = ConvGroupExecution(sess.backend, [l[1] for l in keep])
        st = sess.group.bind([l[2] for l in keep], [l[3] for l in keep])
        assert st == 0, st
        sess.capture()

    rebuild(None)
    alone = split(sess)
    group_b = sum(l[1].cost()[0] for l in members)
    alone.update(group_alg_MB=round(group_b / 1e6, 2), group_hbm_us=round(group_b / PEAK_GBS / 1e3, 2),
                 group_share_of_step=round(alone["group_ms"] / alone["step_ms"], 3))
    full = time_steps(sess)
    rows = []
    for i, (node, ex, x, y) in enumerate(members):
        rebuild(i)
        t = time_steps(sess)
        b, m = ex.cost()
        n, c, h, w = node.attrs["in_shape"]
        rows.append({"layer": i, "name": node.name[-48:], "in": [c, h, w], "out_c": y.shape[1], "alg_MB": round(b / 1e6, 3),
                     "hbm_us": round(b / PEAK_GBS / 1e3, 2), "marginal_us": round((full - t) * 1e3, 2),
                     "frac": round((b / PEAK_GBS / 1e3) / max((full - t) * 1e3, 1e-3), 3)})
    rebuild(None)
    full2 = time_steps(sess)
    print(json.dumps({"device": torch.cuda.get_device_name(), "alone": alone, "full_ms": full, "full_ms_again": full2, "sum_marginal_us": round(sum(r["marginal_us"] for r in rows), 1),
                      "singles": [l[0].name[-40:] for l in sess.singles], "layers": rows}, indent=1))


if __name__ == "__main__":
    main()
