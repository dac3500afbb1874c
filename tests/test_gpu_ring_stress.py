"""-m gpu: the producer / consumer ring of the compositing kernels under maximum pressure.  A second build of the same
sources shrinks the ring to ONE stage of 32 records (gaustudio_b200/build.py::build_stress_variant), so every batch
re-uses the only buffer: a missing wait, a wrong phase parity or an early refill corrupts pixels immediately.  The
stress build must reproduce the default build bit for bit (forward) and to rounding (gradients), and it is also the
build that compute-sanitizer's racecheck / synccheck runs use (tools/sanitize.sh)."""
import json
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STRESS = os.path.join(ROOT, "gaustudio_b200", "libgsr_b200_stress.so")

CHILD = r'''
import sys, json, hashlib, torch
sys.path.insert(0, ".")
from gaustudio_b200 import renderers
from gaustudio_b200.synthetic import build_config
model, cams, c = build_config("cfg2", P=60000, W=400, H=304, K=3)
dev = torch.device("cuda"); model.to(dev).requires_grad_(True)
out = {}
for fused in (False, True):
    r = renderers.make({"name": "vanilla_renderer", "fused_activations": fused})
    for k, cam in enumerate(cams[:2]):
        for p in model.parameters_list(): p.grad = None
        o = r.render(cam.to(dev), model)
        g = torch.Generator().manual_seed(k)
        loss = sum((o[n] * torch.randn(o[n].shape, generator=g).to(dev)).sum() for n in ("render", "rendered_depth", "rendered_final_opacity"))
        loss.backward()
        key = f"{int(fused)}{k}"
        out["img" + key] = hashlib.sha1(torch.cat([o[n].detach().flatten() for n in ("render", "rendered_depth", "rendered_median_depth", "rendered_final_opacity")]).cpu().numpy().tobytes()).hexdigest()
        out["grad" + key] = [float(p.grad.double().abs().sum()) for p in model.parameters_list()]
print("RESULT" + json.dumps(out))
'''


def _run(lib, **extra):
    env = dict(os.environ)
    env.pop("GSR_FWD_TMA", None)
    env.pop("GSR_BWD_NSUB", None)
    if lib:
        env["GSR_LIB"] = lib
    else:
        env.pop("GSR_LIB", None)
    env.update(extra)
    r = subprocess.run([sys.executable, "-c", CHILD], cwd=ROOT, env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    line = [l for l in r.stdout.splitlines() if l.startswith("RESULT")][-1]
    return json.loads(line[6:])


def test_one_stage_ring_reproduces_default_build():
    if not os.path.exists(STRESS):
        pytest.skip("stress variant not built (python -c 'from gaustudio_b200 import build; build.build_stress_variant()')")
    _same(_run(None), _run(STRESS), "with the one-stage ring")  # gradients: float atomics, order-dependent rounding only


def _same(a, b, what):
    for k in a:
        if k.startswith("img"):
            assert a[k] == b[k], f"forward outputs differ {what} ({k})"
        else:
            for x, y in zip(a[k], b[k]):
                assert abs(x - y) <= 1e-5 * max(abs(x), 1e-12), (what, k, x, y)


def test_tma_bulk_staging_reproduces_default_build():
    """GSR_FWD_TMA=1: the compositing forward stages its record batches with TMA bulk copies (one 48-byte cp.async.bulk
    per record, completing on the stage's mbarrier) instead of per-record LDGSTS copies.  Same pixels, bit for bit --
    also on the one-stage ring."""
    ref = _run(None)
    _same(ref, _run(None, GSR_FWD_TMA="1"), "with TMA bulk-copy staging")
    if os.path.exists(STRESS):
        _same(ref, _run(STRESS, GSR_FWD_TMA="1"), "with TMA bulk-copy staging on the one-stage ring")


def test_two_pixels_per_lane_backward_matches_default():
    """GSR_BWD_NSUB=2: every lane owns two pixels (8x8 region per warp) and sums a Gaussian's gradient over both before the
    warp reduction.  Same forward, same gradients up to the order of the float reductions."""
    _same(_run(None), _run(None, GSR_BWD_NSUB="2"), "with two pixels per lane in the backward")
