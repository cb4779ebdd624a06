"""Golden fixtures under tests/golden.

Each fixture is one `torch.save` payload.  Payloads larger than PART_BYTES are stored as consecutive pieces
`<name>.part00`, `<name>.part01`, ... so that no file of the repository exceeds 1 MB; `load` reassembles them."""
from __future__ import annotations

import io
from pathlib import Path

import torch

GOLDEN = Path(__file__).resolve().parent.parent / "tests" / "golden"
PART_BYTES = 1_000_000


def _parts(name: str) -> list[Path]:
    return sorted(GOLDEN.glob(f"{name}.part[0-9][0-9]"))


def save(obj, name: str) -> None:
    buf = io.BytesIO()
    torch.save(obj, buf)
    data = buf.getvalue()
    for old in [GOLDEN / name, *_parts(name)]:
        old.unlink(missing_ok=True)
    if len(data) <= PART_BYTES:
        (GOLDEN / name).write_bytes(data)
        return
    for i in range(0, len(data), PART_BYTES):
        (GOLDEN / f"{name}.part{i // PART_BYTES:02d}").write_bytes(data[i:i + PART_BYTES])


def load(name: str):
    whole = GOLDEN / name
    if whole.exists():
        data = whole.read_bytes()
    else:
        parts = _parts(name)
        if not parts:
            raise FileNotFoundError(f"golden fixture {name} not found under {GOLDEN}")
        data = b"".join(p.read_bytes() for p in parts)
    return torch.load(io.BytesIO(data), map_location="cpu", weights_only=False)
