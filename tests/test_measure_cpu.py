"""scripts/measure.py, the timing scripts' shared helper, without a device: no card means no measurement, and a result
is printed as one JSON line with the card's fields."""
import json
import os
import sys

import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "scripts"))
import measure  # noqa: E402

CARD = dict(card="NVIDIA H100 80GB HBM3", power_limit="700.00 W", sm_clock="1980 MHz", max_sm_clock="1980 MHz")


def test_card_raises_without_a_device(monkeypatch):
    monkeypatch.setattr(measure.torch.cuda, "is_available", lambda: False)
    with pytest.raises(RuntimeError, match="no CUDA device"):
        measure.card()


def test_emit_prints_one_line_with_the_card(monkeypatch, capsys, tmp_path):
    monkeypatch.setattr(measure, "card", lambda: dict(CARD))
    out = tmp_path / "lines.jsonl"
    result = {"ms_call": 1.5, "case": {"grid": [60, 33]}}
    measure.emit(result, str(out))
    lines = capsys.readouterr().out.splitlines()
    assert len(lines) == 1
    assert json.loads(lines[0]) == {**result, **CARD}
    assert out.read_text() == lines[0] + "\n"
