"""Recorded channels without a GPU: the channel table of api.py against the HB_CHANNEL_* macros of the header and their documented element
types and widths, make_channels' shapes and types, and the rejections of hb_rollout_set_channel that need no context."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

import hunter_bipedal_control_b200 as hb

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = open(os.path.join(ROOT, "include", "hunter_b200.h")).read()
TYPES = {"double": np.float64, "int32": np.int32, "uint8": np.uint8}


def test_channel_table_is_the_header():
    doc = re.findall(r"^#define HB_CHANNEL_(\w+) (\d+)\s*/\* (double|int32|uint8) x (\d+)", HEADER, re.M)
    assert len(doc) == len(hb.CHANNELS)
    assert {name.lower(): (int(i), TYPES[t], int(w)) for name, i, t, w in doc} == hb.CHANNELS
    assert int(re.search(r"^#define HB_CHANNELS (\d+)", HEADER, re.M).group(1)) == len(hb.CHANNELS)
    assert sorted(i for i, _, _ in hb.CHANNELS.values()) == list(range(len(hb.CHANNELS)))
    assert "hb_rollout_set_channel" in hb.EXPORTED_SYMBOLS and hasattr(hb.load_library(), "hb_rollout_set_channel")


def test_make_channels_shapes_and_types():
    bufs = hb.make_channels(5, 7, device="cpu")
    assert list(bufs) == list(hb.CHANNELS)
    for name, t in bufs.items():
        _, dtype, width = hb.CHANNELS[name]
        assert t.shape == (5, 7, width) and t.dtype == getattr(torch, np.dtype(dtype).name) and t.is_contiguous() and not t.any()
    some = hb.make_channels(2, 3, ["mode", "contact_flag"], device="cpu")
    assert list(some) == ["mode", "contact_flag"] and some["mode"].dtype == torch.int32 and some["contact_flag"].dtype == torch.uint8
    assert some["contact_flag"].shape == (2, 3, 4)
    with pytest.raises(ValueError, match="unknown channel"):
        hb.make_channels(2, 3, ["torques"], device="cpu")


def test_setter_rejects_without_a_context():
    lib = hb.load_library()
    buf = np.zeros(64)
    p = C.c_void_p(buf.ctypes.data)
    for channel, B, rows, ptr in [(0, 1, 1, p), (0, 0, 0, None), (-1, 1, 1, p), (10, 1, 1, p), (0, -1, 1, p), (0, 1, -1, p), (0, 1, 1, None)]:
        assert lib.hb_rollout_set_channel(None, channel, B, rows, ptr) == -1
