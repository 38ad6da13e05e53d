"""Checkpoints on the SIMT emulator (tests/simt/, with csrc/trl_checkpoint.cu linked into its library here): a miniature of tests/test_gpu_checkpoint.py run without a GPU.  16 envs, 2 training
slots paced by tuples, a replay memory of 160 rows: 3 updates, save, destroy, load, 3 more updates == 6 updates on one handle, under
the permuted lane schedule of the race check (tests/test_simt_cpu.py); the digests of the file against the numpy restatement; a byte
flipped in every section, a truncated file and a wrong version refused with the section or cause named.  As in
tests/test_train_slots_cpu.py, the first tuples of a synchronised start arrive later than an emulator run can afford to wait: the
restored replay memory and the training it drives are compared on the GPU."""
import contextlib
import ctypes as C
import fcntl
import os
import subprocess
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "simt"))
import build as simt_build  # noqa: E402
from test_gpu_checkpoint import PACED, assert_refused, assert_same, check_digests, damaged_copies  # noqa: E402
from test_gpu_train_slots import close, make_group, start_models  # noqa: E402

pytestmark = pytest.mark.skipif(__import__("platform").machine() != "x86_64",
                                reason="the emulator's fiber switch is written for x86-64")
N = 16
TRAINER = dict(replay_mem_size=160, num_init_samples=160, freeze_target_iters=2)
UNIT = "trl_checkpoint.cu"


def checkpoint_build():
    """the emulator library of tests/simt/build.py with the checkpoint unit linked in (its own directory under the emulator's build
    root; the objects of the other units are the default build's)"""
    simt_build.build()
    cdir = os.path.join(simt_build.BUILD_ROOT, "checkpoint")
    os.makedirs(cdir, exist_ok=True)
    out = os.path.join(cdir, "libterrainrl_simt.so")
    csrc = simt_build.CSRC
    deps = [os.path.join(csrc, f) for f in os.listdir(csrc)] + [os.path.join(simt_build.HERE, "simt_runtime.h")]
    deps += [os.path.join(simt_build.HERE, "include", f) for f in os.listdir(os.path.join(simt_build.HERE, "include"))]
    with open(os.path.join(cdir, ".lock"), "w") as lock:
        fcntl.flock(lock, fcntl.LOCK_EX)      # pytest-xdist workers may ask for the same build at the same time
        cxx = os.environ.get("CXX", "g++")
        objs = [os.path.join(simt_build.BUILD_ROOT, "default" if u in simt_build.VARIANT_UNITS else "common", os.path.splitext(u)[0] + ".o")
                for u in simt_build.UNITS + simt_build.LOCAL_UNITS]
        objs += simt_build._compile(cxx, [UNIT], cdir, [], deps, False)
        if not (os.path.exists(out) and all(os.path.getmtime(out) >= os.path.getmtime(o) for o in objs)):
            subprocess.run([cxx, "-shared", "-o", out + ".tmp"] + objs + ["-Wl,--allow-multiple-definition", "-lpthread", "-ldl"], check=True)
            os.replace(out + ".tmp", out)
    return out


@contextlib.contextmanager
def simt_library():
    """the Python mirror pointed at that library for the duration of a test (as tests/simt/loader.py does for the default build)"""
    from deepterrainrl_b200 import scenario
    L = C.CDLL(checkpoint_build())
    L.trl_create_from_pack.restype = C.c_void_p
    L.trl_create_from_pack.argtypes = [C.c_char_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_uint64]
    L.trl_last_error.restype = C.c_char_p
    saved = scenario._LIB
    scenario._LIB = L
    try:
        yield L
    finally:
        scenario._LIB = saved


def test_training_slots_resume_on_the_emulator(assets, tmp_path):
    import deepterrainrl_b200 as trl
    from deepterrainrl_b200.train import TrainSchedule, train_run_slots
    with simt_library() as L:
        pack = os.path.join(assets, "dog_slopes_mixed.trlpack")
        models = start_models(pack, str(tmp_path))[:2]
        slots = np.arange(N) % 2
        scheds = [TrainSchedule(**dict(PACED, init_exp_rate=r)) for r in (0.5, 0.8)]
        L.simt_set_sched_seed(C.c_ulonglong(2024))
        try:
            a, ta = make_group(trl, pack, N, models, slots, trainer_kw=TRAINER)
            b, tb = make_group(trl, pack, N, models, slots, trainer_kw=TRAINER)
            for trs in (ta, tb):
                train_run_slots(trs, scheds, 3, None)
            path = str(tmp_path / "mini.ckpt")
            b.SaveCheckpoint(path, b"mini")
            close(*tb, b)
            b, tb, user = trl.load_checkpoint(path)
            assert user == b"mini" and sorted(tb) == [0, 1]
            tb = [tb[0], tb[1]]
            for trs in (ta, tb):
                train_run_slots(trs, scheds, 3, None)
        finally:
            L.simt_set_sched_seed(C.c_ulonglong(0))
        assert_same(a, b, ta, tb)
        check_digests(path)
        d = tmp_path / "bad"
        d.mkdir()
        for p, msg in damaged_copies(path, str(d)):
            assert_refused(L, p, msg)
        close(*ta, *tb, a, b)
