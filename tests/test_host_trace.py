"""trace_step.py's reading of the dsx_debug_trace slot layout (include/dsx.h), on synthetic stamps."""
import importlib.util
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _trace_step():
    spec = importlib.util.spec_from_file_location("trace_step", os.path.join(ROOT, "trace_step.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def _stamps(ctas, rows, layers, head, barrier_last=True):
    tr = np.zeros((rows, 256), dtype=np.int64)
    for c in range(ctas):
        t = 10_000 + 37 * c
        tr[c, 0] = t
        for i in range(layers):
            for k in range(9):
                if k == 8 and i == layers - 1 and not barrier_last:
                    continue
                t += 1000 * (k + 1)
                tr[c, 1 + 9 * i + k] = t
        for k in range(head):
            t += 500 * (k + 1)
            tr[c, 1 + 9 * layers + k] = t
    return tr


def test_phase_split_with_head():
    ts = _trace_step()
    lay, n, head, nh = ts.phase_split(_stamps(5, 12, 3, 6), 3)
    assert n == 15 and nh == 5
    np.testing.assert_allclose(lay / n, [1, 2, 3, 4, 5, 6, 7, 8, 9])
    np.testing.assert_allclose(head / nh, [0.5, 1.0, 1.5, 2.0, 2.5, 3.0])


def test_phase_split_ignores_stale_head_slots():
    ts = _trace_step()
    tr = _stamps(3, 4, 2, 4)
    tr[:3, 1 + 9 * 2 + 4:1 + 9 * 2 + 6] = 5          # left over from an earlier launch with an input projection
    lay, n, head, nh = ts.phase_split(tr, 2)
    np.testing.assert_allclose(head / nh, [0.5, 1.0, 1.5, 2.0, 0.0, 0.0])


def test_phase_split_last_layer_without_barrier():
    ts = _trace_step()
    lay, n, head, nh = ts.phase_split(_stamps(4, 8, 2, 0, barrier_last=False), 2)
    assert n == 8
    # the missing barrier of the last layer counts as 0 µs
    np.testing.assert_allclose(lay / n, [1, 2, 3, 4, 5, 6, 7, 8, 4.5])
    assert not head.any()
