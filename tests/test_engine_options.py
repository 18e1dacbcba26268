"""Engine switches (MAML_B200_* environment variables): read in one place, documented, and owned by the handle that
read them -- a switch set for one handle must not change what another handle runs."""
import os
import re

import pytest

from conftest import ROOT, load_golden
from engine_layout import rel_err

CSRC = os.path.join(ROOT, "howtotrainyourmamlpytorch_b200", "csrc")
PKG = os.path.join(ROOT, "howtotrainyourmamlpytorch_b200")


def _sources(d, exts):
    return {f: open(os.path.join(d, f)).read() for f in sorted(os.listdir(d)) if f.endswith(exts)}


def _body_span(src, signature):
    """[start, end) of the brace-delimited body of the function whose definition matches `signature`."""
    m = re.search(signature, src)
    assert m, signature
    depth, i = 0, src.index("{", m.start())
    start = i
    while True:
        if src[i] == "{":
            depth += 1
        elif src[i] == "}":
            depth -= 1
            if depth == 0:
                return start, i + 1
        i += 1


def test_getenv_is_called_only_in_read_options():
    srcs = _sources(CSRC, (".cu", ".cuh", ".inc"))
    lo, hi = _body_span(srcs["engine.cu"], r"\bEngineOptions\s+read_options\s*\(\s*\)\s*\{")
    calls = [(f, m.start()) for f, s in srcs.items() for m in re.finditer(r"\bgetenv\s*\(", s)]
    assert calls
    outside = ["%s:%d" % (f, srcs[f].count("\n", 0, p) + 1) for f, p in calls if not (f == "engine.cu" and lo <= p < hi)]
    assert not outside, "getenv outside read_options: %s" % outside


def test_every_switch_is_documented_and_every_documented_switch_exists():
    used = set()
    for s in _sources(CSRC, (".cu", ".cuh", ".inc")).values():
        used |= set(re.findall(r'"MAML_B200_([A-Z0-9_]+)"', s))
    for s in _sources(PKG, (".py",)).values():
        used |= set(re.findall(r'["\']MAML_B200_([A-Z0-9_]+)["\']', s))
    assert {"LIB", "COLLECTIVE"} <= used
    design = open(os.path.join(ROOT, "DESIGN.md")).read()
    table = design[design.index("### Diagnostic switches"):]
    table = table[:table.index("\n\n", table.index("| variable"))]
    documented = set(re.findall(r"^\| `MAML_B200_([A-Z0-9_]+)`", table, flags=re.M))
    assert used == documented, ("undocumented: %s" % sorted(used - documented), "not read anywhere: %s" % sorted(documented - used))


def _model(g, device):
    from howtotrainyourmamlpytorch_b200 import MAMLFewShotClassifier
    a = g.args
    m = MAMLFewShotClassifier(im_shape=(2, a.image_channels, a.image_height, a.image_width), device=device, args=a)
    m.load_state_dict(g.state())
    return m


@pytest.mark.gpu
def test_switches_do_not_leak_between_handles(cuda_device, monkeypatch):
    """Handle B is created with the plain-path switches; handle A (created before) and handle C (created after, with the
    environment restored) must still run the default launch sequence.  Eager launches throughout, so that every call
    enqueues its kernels again and would pick up state left behind by another handle.  A model creates its engine
    handle on its first meta_gradient call."""
    g = load_golden("tiny_pp")
    batch, epoch = g.batch(0), g.iters[0][0]
    monkeypatch.setenv("MAML_B200_NO_GRAPH", "1")
    a = _model(g, cuda_device)
    _, _, grads_a = a.meta_gradient(batch, epoch)
    launches_a = a._engine.last_launch_count()

    with monkeypatch.context() as env:
        for k, v in {"BN_FUSE": "0", "TAIL_FUSE": "0", "TC_SPLIT": "1", "WGRAD_TC": "0"}.items():
            env.setenv("MAML_B200_" + k, v)
        b = _model(g, cuda_device)
        b.meta_gradient(batch, epoch)
        assert b._engine.last_launch_count() != launches_a      # the switches take effect on B

    _, _, grads_a2 = a.meta_gradient(batch, epoch)
    assert a._engine.last_launch_count() == launches_a
    for n in grads_a:
        if "conv.bias" in n or "conv-bias" in n:
            assert float((grads_a2[n] - grads_a[n]).abs().max()) <= 1e-5, n
        else:
            assert rel_err(grads_a2[n], grads_a[n]) <= 2e-5, (n, rel_err(grads_a2[n], grads_a[n]))

    c = _model(g, cuda_device)
    c.meta_gradient(batch, epoch)
    assert c._engine.last_launch_count() == launches_a
