"""GPU clock / throttle sampler for benchmark hygiene: a benchmark reports the clocks its numbers were taken at."""
from __future__ import annotations

import statistics
import subprocess
import threading

_QUERY = (
    "index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.active,"
    "clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
    "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap,utilization.gpu"
)


class ClockSampler:
    """Runs `nvidia-smi --query-gpu=... -lms 200` while a timed region executes."""

    def __init__(self, gpu_index: int = 0, period_ms: int = 200):
        self.gpu_index = gpu_index
        self.period_ms = period_ms
        self._proc = None
        self._lines: list[str] = []
        self._thread = None

    def start(self) -> "ClockSampler":
        try:
            self._proc = subprocess.Popen(
                ["nvidia-smi", f"--query-gpu={_QUERY}", "--format=csv,noheader,nounits", "-lms", str(self.period_ms),
                 "-i", str(self.gpu_index)],
                stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
        except OSError:
            self._proc = None
            return self

        def pump():
            assert self._proc is not None and self._proc.stdout is not None
            for line in self._proc.stdout:
                self._lines.append(line.strip())

        self._thread = threading.Thread(target=pump, daemon=True)
        self._thread.start()
        return self

    def stop(self) -> dict:
        if self._proc is not None:
            self._proc.terminate()
            try:
                self._proc.wait(timeout=2)
            except subprocess.TimeoutExpired:
                self._proc.kill()
        if self._thread is not None:
            self._thread.join(timeout=2)
        sm, smax, busy, reasons = [], [], [], set()
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        for line in self._lines:
            parts = [p.strip() for p in line.split(",")]
            if len(parts) < 9:
                continue
            try:
                sm.append(float(parts[1]))
                smax.append(float(parts[2]))
            except ValueError:
                continue
            try:  # samples taken while kernels were resident: the idle stretches of a multi-phase run (cluster bring-up,
                if len(parts) > 9 and float(parts[9]) > 0:  # rendezvous, host-side verification) sit at the idle clock
                    busy.append(sm[-1])
            except ValueError:
                pass
            for name, val in zip(names, parts[5:9]):
                if val.lower().startswith("active"):
                    reasons.add(name)
        return {
            "sm_mhz": statistics.median(busy) if busy else (statistics.median(sm) if sm else None),
            "sm_max_mhz": max(smax) if smax else None,
            "samples": len(sm),
            "samples_under_load": len(busy),
            "sm_mhz_all_samples": statistics.median(sm) if sm else None,
            "reasons": sorted(reasons),
        }
