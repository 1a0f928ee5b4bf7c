"""Config 5 in miniature for the decoder: 1 KiB records compressed against one 16 KiB dictionary, decoded one call per record.
Per-call time of ZSTD_decompress_usingDict (the dictionary digested and uploaded by every call) against a resident DDict
(ZSTD_decompress_usingDDict for host buffers, a sticky DDict with ZSTDB200_decompressDevice for device buffers), with the
card's name and power limit.  Needs a GPU.

    python tests/bench_ddict.py [--records 2000] [--rounds 3] [--out /tmp/bench_ddict.json]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import zref  # noqa: E402
import zstd_b200  # noqa: E402

_sz, _vp = ctypes.c_size_t, ctypes.c_void_p


def card():
    name = torch.cuda.get_device_name(0)
    try:
        power = subprocess.check_output(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], text=True).strip()
    except (OSError, subprocess.CalledProcessError):
        power = "unknown"
    return name, power


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--records", type=int, default=2000)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    L = zstd_b200.lib()
    L.ZSTD_decompress_usingDict.restype = _sz
    L.ZSTD_decompress_usingDict.argtypes = [_vp, _vp, _sz, _vp, _sz, _vp, _sz]
    L.ZSTDB200_decompressDevice_usingDict.restype = _sz
    L.ZSTDB200_decompressDevice_usingDict.argtypes = [_vp, _vp, _sz, _vp, _sz, _vp, _sz, _vp]
    d = zref.golden_input("zdict-16k-synthetic-seed77")
    cctx = zstd_b200.ZSTD_CCtx()
    recs = [zref.synthetic(1024, 1000 + i, 0.5) for i in range(a.records)]
    frames = [cctx.compress_using_dict(r, d, 1) for r in recs]
    dctx = zstd_b200.ZSTD_DCtx()
    dd = zstd_b200.ZSTD_DDict(d)
    out = ctypes.create_string_buffer(1024)
    d_in = [torch.frombuffer(bytearray(f), dtype=torch.uint8).cuda() for f in frames]
    d_out = torch.empty(1024, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()

    def host_dict():
        for f in frames:
            assert L.ZSTD_decompress_usingDict(dctx._h, out, 1024, f, len(f), d, len(d)) == 1024

    def host_ddict():
        for f in frames:
            assert L.ZSTD_decompress_usingDDict(dctx._h, out, 1024, f, len(f), dd._h) == 1024

    def device_dict():
        for x in d_in:
            assert L.ZSTDB200_decompressDevice_usingDict(dctx._h, d_out.data_ptr(), 1024, x.data_ptr(), x.numel(), d, len(d), None) == 1024

    def device_ddict():
        for x in d_in:
            assert L.ZSTDB200_decompressDevice(dctx._h, d_out.data_ptr(), 1024, x.data_ptr(), x.numel(), None) == 1024

    def sticky(fn):
        def run():
            dctx.ref_ddict(dd)
            try:
                fn()
            finally:
                dctx.ref_ddict(None)
        return run
    cases = {"host usingDict": host_dict, "host usingDDict": host_ddict, "device usingDict": device_dict,
             "device sticky DDict": sticky(device_ddict)}
    for fn in cases.values():                                        # warm-up: buffers grown, the DDict resident
        fn()
    us = {k: [] for k in cases}
    for _ in range(a.rounds):                                        # alternating, so that drift hits every case alike
        for k, fn in cases.items():
            t = time.perf_counter()
            fn()
            us[k].append((time.perf_counter() - t) / a.records * 1e6)
    assert dctx.decompress_using_ddict(frames[0], dd) == recs[0]
    name, power = card()
    res = {"gpu": name, "power_limit": power, "records": a.records, "record_bytes": 1024, "dict_bytes": len(d),
           "us_per_call": {k: [round(x, 1) for x in v] for k, v in us.items()}}
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
