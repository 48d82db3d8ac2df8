"""Developer tool: where the time of hg_compact_to_sst goes, per page codec.  The inputs of tools/bench_compaction.py (k overlapping SSTs,
resident in HBM) are compacted to an SST with codec none / snappy / zstd, and with DELTA_BINARY_PACKED / dictionary pages (Snappy: keys
`delta_ints_snappy`, `dict_keys_snappy`, `mixed_snappy`), under torch.profiler (CUDA activities); prints one JSON line
with the device time per kernel name, summed over `reps` calls and divided by `reps`, plus the card's name and power limit.

Usage: profile_sst_writer.py [k=16] [series=4000] [points=1000] [keep=0.5] [reps=3]"""
import json
import os
import subprocess
import sys
import tempfile
from collections import defaultdict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

k = int(sys.argv[1]) if len(sys.argv) > 1 else 16
series = int(sys.argv[2]) if len(sys.argv) > 2 else 4000
points = int(sys.argv[3]) if len(sys.argv) > 3 else 1000
keep = float(sys.argv[4]) if len(sys.argv) > 4 else 0.5
reps = int(sys.argv[5]) if len(sys.argv) > 5 else 3

if __name__ == "__main__":
    import torch
    from torch.profiler import ProfilerActivity, profile

    from horaedb_b200 import sstgen
    from horaedb_b200._ffi import Engine, SchemaHandle, SstInput

    schema = sstgen.metric_storage_schema()
    handle = SchemaHandle(schema.arrow_schema, 2)
    eng = Engine(device=0)
    inputs = []
    for f in range(k):
        data, n, seq = sstgen.synth_overlapping_ssts(1, series, points, 1000, keep, base_seq=1000 + f)[0]
        eng.load_sst(handle, SstInput(id=seq, data=data, num_rows=n))
        inputs.append(SstInput(id=seq, num_rows=n, time_start=0, time_end=1, max_sequence=seq))
    path = os.path.join(tempfile.mkdtemp(), "out.sst")
    torch.cuda.init()
    from horaedb_b200.config import ColumnOptions, WriteConfig, resolve_column_options
    D = "DELTA_BINARY_PACKED"
    runs = {codec: {"compression": codec} for codec in ("none", "snappy", "zstd")}
    for name, wcfg in (("delta_ints_snappy", WriteConfig(encoding=D, column_options={"value": ColumnOptions(encoding="PLAIN")})),
                       ("dict_keys_snappy", WriteConfig(column_options={n: ColumnOptions(enable_dict=True) for n in ("series_id", "tag", "__seq__")})),
                       ("mixed_snappy", WriteConfig(column_options={"series_id": ColumnOptions(enable_dict=True), "tag": ColumnOptions(enable_dict=True),
                                                                    "ts": ColumnOptions(encoding=D), "__seq__": ColumnOptions(encoding=D)}))):
        runs[name] = {"columns": resolve_column_options(wcfg, schema.arrow_schema)}
    out = {}
    for codec, kw in runs.items():
        eng.compact_to_sst(handle, inputs, path, **kw)                              # warm-up
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(reps):
                eng.compact_to_sst(handle, inputs, path, **kw)
        per = defaultdict(float)
        for ev in prof.events():
            if ev.device_type == torch.autograd.DeviceType.CUDA:
                name = ev.name.replace("(anonymous namespace)::", "").replace("horae::", "").replace("void ", "").split("(")[0].split("<")[0]
                per[name] += ev.device_time_total / 1e3 / reps
        out[codec] = {"kernels_ms": dict(sorted(per.items(), key=lambda kv: -kv[1])), "total_ms": sum(per.values())}
    eng.close()
    try:
        gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.TimeoutExpired):
        gpu = "unknown"
    print(json.dumps({"gpu": gpu, "reps": reps, "by_codec": out}))
