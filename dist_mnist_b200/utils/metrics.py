"""Measurement helpers: GPU clock/throttle sampling during a timed region, CUDA-event timing.

The reference measures nothing (no timers anywhere in /root/reference — SURVEY §5 "Tracing / profiling");
the metric of this repo is device-timed steps/sec, so this module is new-build only. The clock sampler follows
the profiling recipe: `nvidia-smi --query-gpu=... -lms 200` started before the timed region, stopped after,
summarised as the median SM clock under load plus the set of throttle reasons that were active.
"""
from __future__ import annotations

import csv
import io
import json
import shutil
import statistics
import subprocess
import tempfile
import time
from typing import Dict, List, Optional

import contextlib
import functools

import torch

_QUERY = ("index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.active,"
          "clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
          "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")


class ClockSampler:
    """Samples nvidia-smi in a subprocess between start() and stop()."""

    def __init__(self, interval_ms: int = 100, gpu_indices: Optional[List[int]] = None):
        self.interval_ms = interval_ms
        self.gpu_indices = gpu_indices
        self._proc = None
        self._out = None

    def start(self) -> None:
        if shutil.which("nvidia-smi") is None:
            return
        self._out = tempfile.NamedTemporaryFile(mode="w+", suffix=".csv", delete=False)
        cmd = ["nvidia-smi", f"--query-gpu={_QUERY}", "--format=csv,noheader,nounits", "-lms", str(self.interval_ms)]
        if self.gpu_indices:
            cmd += ["-i", ",".join(str(i) for i in self.gpu_indices)]
        try:
            self._proc = subprocess.Popen(cmd, stdout=self._out, stderr=subprocess.DEVNULL)
        except Exception:
            self._proc = None

    def stop(self) -> Dict:
        if self._proc is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": [], "samples": 0}
        time.sleep(self.interval_ms / 1000.0)
        self._proc.terminate()
        try:
            self._proc.wait(timeout=5)
        except Exception:
            self._proc.kill()
        self._out.flush()
        self._out.seek(0)
        text = self._out.read()
        self._out.close()
        return summarize_clock_csv(text)


def summarize_clock_csv(text: str) -> Dict:
    sm, smax, power = [], [], []
    reasons = set()
    names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
    for row in csv.reader(io.StringIO(text)):
        row = [c.strip() for c in row]
        if len(row) < 9:
            continue
        try:
            sm.append(float(row[1]))
            smax.append(float(row[2]))
            power.append(float(row[3]))
        except ValueError:
            continue
        for name, val in zip(names, row[5:9]):
            if val.lower().startswith("active"):
                reasons.add(name)
    if not sm:
        return {"sm_mhz": None, "sm_max_mhz": None, "reasons": [], "samples": 0}
    return {
        "sm_mhz": statistics.median(sm),
        "sm_max_mhz": max(smax),
        "power_w_max": max(power) if power else None,
        "reasons": sorted(reasons),
        "samples": len(sm),
    }


class StreamTimer:
    """CUDA-event timer on an arbitrary (raw) stream."""

    def __init__(self, stream_ptr: int, device: int):
        self.stream = torch.cuda.ExternalStream(stream_ptr, device=device)
        self.t0 = torch.cuda.Event(enable_timing=True)
        self.t1 = torch.cuda.Event(enable_timing=True)

    def start(self) -> None:
        self.t0.record(self.stream)

    def stop(self) -> None:
        self.t1.record(self.stream)

    def elapsed_ms(self) -> float:
        self.t1.synchronize()
        return self.t0.elapsed_time(self.t1)


class TrainMetricsWriter:
    """The reference's implicit `StepCounterHook` / `SummarySaverHook` (MonitoredTrainingSession defaults, SURVEY
    §3.4): every `every_steps` local steps one JSON line {time, worker, local_steps, global_step, loss,
    batch_accuracy, steps_per_sec} is appended to `path` (accuracy comes for free: the head kernel counts the
    correct predictions of every training batch), and optionally an INFO-style `global_step/sec` line is printed.
    `lr_at` (a learning-rate schedule, global step -> rate) adds the rate at the line's global step as
    `learning_rate`, like the learning-rate summary of a TF1 script."""

    def __init__(self, path: Optional[str], worker_index: int, batch_size: int, every_steps: int = 100,
                 echo: bool = False, print_fn=print, lr_at=None):
        self.path, self.worker, self.batch, self.every, self.echo, self.print_fn = (
            path, worker_index, batch_size, max(1, every_steps), echo, print_fn)
        self.lr_at = lr_at
        self._fh = open(path, "a") if path else None
        self._t_last = time.time()
        self._steps = 0
        self._steps_last = 0
        self._gs_last: Optional[int] = None
        self._loss_sum = 0.0
        self._correct = 0
        self._n = 0

    def update(self, outs) -> None:
        """Feed the results of a run of steps (any sequence of StepOutput)."""
        for o in outs:
            self._steps += 1
            self._loss_sum += o.loss
            self._correct += o.correct
            self._n += 1
            if self._steps - self._steps_last >= self.every:
                self._emit(o.global_step)

    def _emit(self, global_step: int) -> None:
        now = time.time()
        dt = max(now - self._t_last, 1e-9)
        rec = {
            "time": round(now, 3), "worker": self.worker, "local_steps": self._steps, "global_step": int(global_step),
            "loss": self._loss_sum / max(self._n, 1),
            "batch_accuracy": self._correct / max(self._n * self.batch, 1),
            "steps_per_sec": (self._steps - self._steps_last) / dt,
        }
        if self._gs_last is not None:
            rec["global_steps_per_sec"] = (int(global_step) - self._gs_last) / dt
        if self.lr_at is not None:
            rec["learning_rate"] = self.lr_at(int(global_step))
        if self._fh:
            self._fh.write(json.dumps(rec) + "\n")
            self._fh.flush()
        if self.echo:
            self.print_fn("INFO global_step/sec: {:.1f} (this worker {:.1f} steps/sec, batch accuracy {:.3f})".format(
                rec.get("global_steps_per_sec", rec["steps_per_sec"]), rec["steps_per_sec"], rec["batch_accuracy"]))
        self._t_last, self._steps_last, self._gs_last = now, self._steps, int(global_step)
        self._loss_sum, self._correct, self._n = 0.0, 0, 0

    def close(self) -> None:
        if self._fh:
            self._fh.close()
            self._fh = None


_NVTX = None


def _nvtx():
    global _NVTX
    if _NVTX is None:
        try:
            ok = torch.cuda.is_available()
            from torch.cuda import nvtx as mod
            _NVTX = mod if ok else False
        except Exception:
            _NVTX = False
    return _NVTX


@contextlib.contextmanager
def nvtx_range(name: str):
    """NVTX range around a host-side phase (SURVEY A1; the native runtime adds its own ranges, csrc/trace.h). A push /
    pop is a host-only call into the NVTX shim — no CUDA synchronisation, safe next to a resident persistent kernel —
    and a no-op on a machine without CUDA."""
    global _NVTX
    m = _nvtx()
    if m:
        try:
            m.range_push(name)
        except Exception:   # an unusable NVTX shim must never take training down: switch tracing off
            _NVTX = m = False
    if not m:
        yield
        return
    try:
        yield
    finally:
        try:
            m.range_pop()
        except Exception:
            _NVTX = False


def nvtx_annotate(name: str):
    """Decorator form of nvtx_range."""
    def deco(fn):
        @functools.wraps(fn)
        def wrapped(*a, **kw):
            with nvtx_range(name):
                return fn(*a, **kw)
        return wrapped
    return deco
