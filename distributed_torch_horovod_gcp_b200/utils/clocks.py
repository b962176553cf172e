"""Background sampler of SM clocks / throttle reasons during a timed region (bench.py
``"clocks"`` key).  Uses NVML in a
thread; falls back to ``nvidia-smi`` polling; never changes clocks."""
from __future__ import annotations

import statistics
import subprocess
import threading
from typing import Dict, List, Optional

_REASONS = {
    0x1: "gpu_idle", 0x2: "applications_clocks_setting", 0x4: "sw_power_cap",
    0x8: "hw_slowdown", 0x10: "sync_boost", 0x20: "sw_thermal_slowdown",
    0x40: "hw_thermal_slowdown", 0x80: "hw_power_brake_slowdown", 0x100: "display_clock_setting",
}


class ClockSampler:
    def __init__(self, device_index: int = 0, interval_s: float = 0.1):
        self.idx, self.interval = device_index, interval_s
        self._stop = threading.Event()
        self._thr: Optional[threading.Thread] = None
        self.sm: List[int] = []
        self.reasons = set()
        self.sm_max = 0
        self.power_max = 0.0
        self._mode = None

    def _loop_nvml(self):
        import pynvml
        h = pynvml.nvmlDeviceGetHandleByIndex(self.idx)
        try:
            self.sm_max = pynvml.nvmlDeviceGetMaxClockInfo(h, pynvml.NVML_CLOCK_SM)
        except Exception:
            self.sm_max = 0
        while not self._stop.is_set():
            try:
                self.sm.append(pynvml.nvmlDeviceGetClockInfo(h, pynvml.NVML_CLOCK_SM))
                r = pynvml.nvmlDeviceGetCurrentClocksEventReasons(h) \
                    if hasattr(pynvml, "nvmlDeviceGetCurrentClocksEventReasons") \
                    else pynvml.nvmlDeviceGetCurrentClocksThrottleReasons(h)
                for bit, nm in _REASONS.items():
                    if r & bit and nm not in ("gpu_idle",):
                        self.reasons.add(nm)
                try:
                    self.power_max = max(self.power_max, pynvml.nvmlDeviceGetPowerUsage(h) / 1e3)
                except Exception:
                    pass
            except Exception:
                pass
            self._stop.wait(self.interval)

    def _loop_smi(self):
        q = ("clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,"
             "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,"
             "clocks_event_reasons.sw_power_cap")
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        while not self._stop.is_set():
            try:
                out = subprocess.run(
                    ["nvidia-smi", f"--id={self.idx}", f"--query-gpu={q}",
                     "--format=csv,noheader,nounits"], capture_output=True, text=True,
                    timeout=5).stdout.strip().split(",")
                self.sm.append(int(float(out[0])))
                self.sm_max = int(float(out[1]))
                try:
                    self.power_max = max(self.power_max, float(out[2]))
                except ValueError:
                    pass
                for nm, v in zip(names, out[3:]):
                    if v.strip().lower().startswith("active"):
                        self.reasons.add(nm)
            except Exception:
                pass
            self._stop.wait(max(self.interval, 0.2))

    def start(self):
        try:
            import pynvml
            pynvml.nvmlInit()
            target = self._loop_nvml
            self._mode = "nvml"
        except Exception:
            target = self._loop_smi
            self._mode = "nvidia-smi"
        self._thr = threading.Thread(target=target, daemon=True)
        self._thr.start()
        return self

    def stop(self) -> Dict:
        self._stop.set()
        if self._thr is not None:
            self._thr.join(timeout=5)
        return {
            "sm_mhz": int(statistics.median(self.sm)) if self.sm else None,
            "sm_max_mhz": self.sm_max or None,
            "reasons": sorted(self.reasons),
            "samples": len(self.sm),
            "power_w_max": round(self.power_max, 1) if self.power_max else None,
            "source": self._mode,
        }
