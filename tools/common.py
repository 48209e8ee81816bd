"""What every measurement tool here reads beside its numbers: the card the run is on, and the host-clock timer."""
import subprocess
import time

import torch


def card():
    """Name, power limit and SM clocks of the current CUDA device, read by one read-only nvidia-smi query in the same run as
    the measurement.  The fields are in nvidia-smi's order, so ", ".join(card().values()) is its CSV line."""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=index,name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        dev = str(torch.cuda.current_device())
        row = [r for r in out if r.split(",")[0].strip() == dev] or out
        _, name, power, sm, max_sm = [c.strip() for c in row[0].split(",")]
        return {"name": name, "power_limit": power, "sm_clock": sm, "max_sm_clock": max_sm}
    except (OSError, ValueError, IndexError, subprocess.SubprocessError) as e:
        return {"name": torch.cuda.get_device_name(), "power_limit": "unknown (%s)" % e, "sm_clock": "unknown",
                "max_sm_clock": "unknown"}


def timed(fn):
    """(seconds, fn()) on the host clock, the device synchronised before and after: the time of everything fn queues."""
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out
