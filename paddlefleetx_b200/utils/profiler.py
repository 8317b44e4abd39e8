"""Step-windowed profiler (reference ppfleetx/core/engine/eager_engine.py:223-251 & :776-813 wraps paddle.profiler with a
``scheduler: [start, end]`` window and prints summary views).

B200-first design: the primary signal is *device time per kernel* from CUPTI via ``torch.profiler`` restricted to the scheduled
step window, plus NVTX ranges (``torch.cuda.nvtx``) around every step so that an external ``ncu --nvtx`` capture can be aligned
with the same window.  The summary is written both as a chrome trace and as a flat per-kernel table (json) under
``profiler_log``.
"""
from __future__ import annotations

import json
import os

import torch

from .log import logger


class StepProfiler:
    def __init__(self, cfg):
        sched = cfg.get("scheduler", [1, 5])
        self.start, self.end = int(sched[0]), int(sched[1])
        self.log_dir = cfg.get("profiler_log", "profiler_log")
        self.detailed = bool(cfg.get("detailed", False))
        self.record_shapes = bool(cfg.get("record_shapes", True))
        self.profile_memory = bool(cfg.get("profile_memory", True))
        self._step = 0
        self._prof = None
        self._range_open = False
        self._finished = False
        os.makedirs(self.log_dir, exist_ok=True)
        self._open_range()

    def _open_range(self):
        if torch.cuda.is_available():
            torch.cuda.nvtx.range_push(f"train_step_{self._step}")
            self._range_open = True

    def _close_range(self):
        if self._range_open:
            torch.cuda.nvtx.range_pop()
            self._range_open = False

    def _start(self):
        acts = [torch.profiler.ProfilerActivity.CPU]
        if torch.cuda.is_available():
            acts.append(torch.profiler.ProfilerActivity.CUDA)
        self._prof = torch.profiler.profile(activities=acts, record_shapes=self.record_shapes,
                                            profile_memory=self.profile_memory, with_stack=self.detailed)
        self._prof.__enter__()

    def _stop(self):
        if self._prof is None:
            return
        self._prof.__exit__(None, None, None)
        prof, self._prof = self._prof, None
        rank = int(os.environ.get("RANK", 0))
        try:
            prof.export_chrome_trace(os.path.join(self.log_dir, f"trace_rank{rank}.json"))
        except Exception as exc:  # pragma: no cover
            logger.warning(f"chrome trace export failed: {exc}")
        rows = []
        for ev in prof.key_averages():
            dev = getattr(ev, "device_time_total", getattr(ev, "cuda_time_total", 0.0))
            rows.append({"name": ev.key, "count": ev.count, "cpu_us": ev.cpu_time_total, "device_us": dev})
        rows.sort(key=lambda r: -(r["device_us"] or r["cpu_us"]))
        with open(os.path.join(self.log_dir, f"summary_rank{rank}.json"), "w") as f:
            json.dump({"window": [self.start, self.end], "events": rows[:200]}, f, indent=1)
        sort_key = "self_cuda_time_total" if torch.cuda.is_available() else "self_cpu_time_total"
        logger.info("profiler summary (steps %d..%d):\n%s" % (self.start, self.end, prof.key_averages().table(sort_by=sort_key, row_limit=25)))

    def step(self):
        """Called once at the end of every train step."""
        self._close_range()
        self._step += 1
        if self._step == self.start and self._prof is None and not self._finished:
            self._start()
        elif self._step == self.end and self._prof is not None:
            self._stop()
            self._finished = True
        self._open_range()

    def finish(self):
        self._close_range()
        if self._prof is not None:
            self._stop()
        self._finished = True
