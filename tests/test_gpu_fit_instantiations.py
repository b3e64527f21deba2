"""
A census of the Dense fit kernels: every instantiation of ffae_fit_kernel<WG, DG, SPLIT, STOP, LOSS, OPT> that launch_fit
(csrc/ffae_fit.cu) dispatches to runs, one tiny launch per (memory plan group, entry point, kernel family), the kernel names read
back with torch.profiler.  A template flag added later fails the census until a launch here reaches its kernels.
"""
import re

import numpy as np
import pytest
from parity_helpers import FIT_KW
from test_fit_plan import PLAN_SHAPES

pytestmark = pytest.mark.gpu

# launch_fit's dispatch, as data.  (WG, DG) from the memory plan: everything in shared memory, the weight image in L2, and one to three
# dz buffers in L2 as well (one instantiation for all three), each with a PLAN_SHAPES shape.  (SPLIT, STOP) from the entry point:
# gb_ffae_fit, gb_ffae_fit_split, gb_ffae_fit_stop (gb_ffae_fit_opt takes the one its split and stop arguments name).  (LOSS, OPT) from
# the family: MSE with Adam, another loss, another optimizer than plain Adam (instantiated with LOSS only).
PLAN_GROUPS = {(False, False): (0, 0), (True, False): (1, 0), (True, True): (1, 1)}
ENTRIES = {"fit": (False, False), "split": (True, False), "stop": (True, True)}
FAMILIES = {"mse-adam": (False, False), "huber-adam": (True, False), "mae-nadam": (True, True)}
EXPECTED = {group + entry + family for group in PLAN_GROUPS for entry in ENTRIES.values() for family in FAMILIES.values()}


def template_flags(kernel_name):
    """The six booleans of an ffae_fit_kernel name, demangled (`ffae_fit_kernel<true, false, ...>`) or mangled (`ffae_fit_kernelILb1E...`)."""
    m = re.search(r"ffae_fit_kernel<([^>]*)>", kernel_name)
    if m:
        return tuple(a.strip() == "true" for a in m.group(1).split(","))
    m = re.search(r"ffae_fit_kernelI((?:Lb[01]E)+)", kernel_name)
    return tuple(b == "1" for b in re.findall(r"Lb([01])E", m.group(1))) if m else None


def test_every_fit_kernel_instantiation_runs():
    import torch

    if not torch.cuda.is_available():
        pytest.skip("needs an H100")
    import __graft_entry__ as ge

    ge.build()
    from torch.profiler import ProfilerActivity, profile

    from gordo_components_b200 import engine

    assert len(EXPECTED) == 27
    N, NV = 40, 8
    launches = 0
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for plan in PLAN_GROUPS.values():
            spec = PLAN_SHAPES[plan]
            eng = engine.FFEngine(spec.dims, spec.acts, spec.l1)
            x = torch.from_numpy(np.random.default_rng(0).random((N + NV, spec.dims[0]), dtype=np.float32)).to(eng.device)
            jobs = engine.jobs_to_device(engine.make_jobs([0], [N], [0]), eng.device)
            split = engine.make_split([NV])
            for entry in ENTRIES:
                for family in FAMILIES:
                    p = torch.zeros((1, eng.param_stride), dtype=torch.float32, device=eng.device)
                    kw = dict(epochs=1, batch_size=32, **FIT_KW[family])
                    if entry == "fit":
                        eng.fit(p, jobs, 1, N, x, x, **kw)
                    else:
                        stop = engine.make_stop([{"monitor": "loss", "patience": 1}]) if entry == "stop" else None
                        eng.fit_split(p, jobs, 1, N, x, x, split=split, stop=stop, **kw)
                    launches += 1
        torch.cuda.synchronize()
    names = [e.key for e in prof.key_averages() if "ffae_fit_kernel" in e.key]
    if not names:
        pytest.skip("the profiler lists no kernels here")
    seen = {template_flags(k) for k in names}
    assert None not in seen, names
    assert launches == len(EXPECTED)
    assert seen == EXPECTED, (sorted(EXPECTED - seen), sorted(seen - EXPECTED))
