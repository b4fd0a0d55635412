"""Golden vectors under tests/golden/, kept below 1 MB per file.

``save`` packs a dict of arrays into ``<name>.npz`` plus, when the compressed total would exceed the limit,
``<name>.part<k>.npz`` files; an array that alone exceeds the limit is split along axis 0 into keys ``<key>#<i>``.
``load`` reassembles the dict bit for bit, so every test compares against exactly the values that were minted."""
from __future__ import annotations

import glob
import io
import os
import re

import numpy as np

LIMIT = 1_000_000


def _packed_size(arrays: dict) -> int:
    buf = io.BytesIO()
    np.savez_compressed(buf, **arrays)
    return buf.tell()


def save(golden_dir: str, name: str, limit: int = LIMIT, **arrays) -> list[str]:
    pieces: list[tuple[str, np.ndarray]] = []
    for key, a in arrays.items():
        a = np.asarray(a)
        n = 1
        while a.ndim and _packed_size({key: a[: -(-a.shape[0] // n)]}) > 0.9 * limit and n < a.shape[0]:
            n *= 2
        if n == 1:
            pieces.append((key, a))
        else:
            for i, part in enumerate(np.array_split(a, n, axis=0)):
                pieces.append((f"{key}#{i}", part))
    parts: list[dict] = [{}]
    for key, a in pieces:
        if parts[-1] and _packed_size({**parts[-1], key: a}) > limit:
            parts.append({})
        parts[-1][key] = a
    for old in glob.glob(os.path.join(golden_dir, f"{name}.part*.npz")):
        os.remove(old)
    paths = []
    for k, part in enumerate(parts):
        path = os.path.join(golden_dir, f"{name}.npz" if k == 0 else f"{name}.part{k}.npz")
        np.savez_compressed(path, **part)
        paths.append(path)
    return paths


def load(golden_dir: str, name: str) -> dict:
    out: dict = {}
    split: dict = {}
    paths = [os.path.join(golden_dir, f"{name}.npz")]
    paths += sorted(glob.glob(os.path.join(golden_dir, f"{name}.part*.npz")),
                    key=lambda p: int(re.search(r"\.part(\d+)\.npz$", p).group(1)))
    for path in paths:
        with np.load(path) as z:
            for key in z.files:
                m = re.fullmatch(r"(.+)#(\d+)", key)
                if m:
                    split.setdefault(m.group(1), {})[int(m.group(2))] = z[key]
                else:
                    out[key] = z[key]
    for key, chunks in split.items():
        out[key] = np.concatenate([chunks[i] for i in range(len(chunks))], axis=0)
    return out
