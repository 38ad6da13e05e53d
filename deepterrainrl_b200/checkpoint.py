"""Resume a run from a checkpoint (trl_create_from_checkpoint): the scenario and its trainers as they were when
BatchedScenario.SaveCheckpoint wrote the file.  Every later call on them returns, bit for bit, what the same call returns on the
objects that saved it."""
import ctypes as C
import os
import struct

import numpy as np

from .scenario import ScenarioExpMACE, ScenarioPoliEval, load_library
from .trainer import MACETrainer

MAGIC = b"TRLCKPT1"
SECTION = struct.Struct("<48sIIQQ")      # name, dtype, kind, bytes, digest (csrc/trl_checkpoint.cu: FileSection)


def sections(path):
    """the section table of a checkpoint file: [(name, dtype, kind, offset, bytes, digest)] in file order"""
    with open(path, "rb") as f:
        head = f.read(16)
        if len(head) < 16 or head[:8] != MAGIC:
            raise ValueError(f"{path}: not a checkpoint")
        _, count = struct.unpack("<II", head[8:])
        table = f.read(count * SECTION.size)
    out, off = [], 16 + count * SECTION.size
    for k in range(count):
        name, dtype, kind, nbytes, digest = SECTION.unpack_from(table, k * SECTION.size)
        out.append((name.split(b"\0", 1)[0].decode(), dtype, kind, off, nbytes, digest))
        off += nbytes
    return out


def load_checkpoint(path, device=0):
    """(scenario, {slot: MACETrainer}, user_bytes): the scenario is a ScenarioPoliEval or a ScenarioExpMACE after the stored mode"""
    L = load_library()
    L.trl_create_from_checkpoint.restype = C.c_void_p
    L.trl_create_from_checkpoint.argtypes = [C.c_char_p, C.c_int, C.c_void_p, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]
    table = {s[0]: s for s in sections(path)}
    if "user" not in table or "meta" not in table:
        raise RuntimeError(f"{path}: a checkpoint without its user or meta section")
    with open(path, "rb") as f:
        f.seek(table["meta"][3])
        mode = struct.unpack("<ii", f.read(8))[1]        # Meta: n, mode
    trainers = (C.c_void_p * 8)()
    n_user = C.c_size_t(0)
    user = C.create_string_buffer(max(1, table["user"][4]))
    h = L.trl_create_from_checkpoint(os.fspath(path).encode(), int(device), trainers, user, len(user), C.byref(n_user))
    if not h:
        raise RuntimeError(L.trl_last_error().decode())
    sc = (ScenarioExpMACE if mode == 1 else ScenarioPoliEval)._wrap(L, h)
    trs = {p: MACETrainer._wrap(sc, trainers[p]) for p in range(8) if trainers[p]}
    slots = np.zeros(sc.num_envs, np.int32)
    sc._ck(L.trl_env_policy(sc.h, slots.ctypes.data_as(C.c_void_p), sc.num_envs))
    if slots.any():
        sc._env_slot = slots
    return sc, trs, user.raw[:n_user.value]
