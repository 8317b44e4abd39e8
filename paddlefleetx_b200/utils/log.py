"""Rank-aware colour logger with the two extra levels the trainer uses.

Behavioural parity with the reference logger (ppfleetx/utils/log.py:33-189):
  * extra levels ``TRAIN`` (21) and ``EVAL`` (22) between INFO and WARNING,
  * an ``advertise()`` banner printed before the config dump,
  * ``get_timestamp()`` = device-synchronise, then wall clock; this is what the
    ``avg_batch_cost`` / ``ips`` fields of the canonical train line are built on.

The implementation is a plain ``logging`` tree: one ``StreamHandler`` with an ANSI
formatter, no third-party colour packages.
"""
from __future__ import annotations

import contextlib
import datetime
import logging
import os
import sys
import threading
import time

TRAIN_LEVEL = 21
EVAL_LEVEL = 22
logging.addLevelName(TRAIN_LEVEL, "TRAIN")
logging.addLevelName(EVAL_LEVEL, "EVAL")

_ANSI = {
    "DEBUG": "\033[35m",
    "INFO": "\033[0m",
    "TRAIN": "\033[36m",
    "EVAL": "\033[34m",
    "WARNING": "\033[33m",
    "ERROR": "\033[31m",
    "CRITICAL": "\033[1;31m",
}
_RESET = "\033[0m"


class _AnsiFormatter(logging.Formatter):
    def __init__(self, use_color: bool):
        super().__init__("[%(asctime)s] [%(levelname)8s] - %(message)s", "%Y-%m-%d %H:%M:%S")
        self._color = use_color

    def format(self, record: logging.LogRecord) -> str:
        text = super().format(record)
        if self._color:
            return f"{_ANSI.get(record.levelname, '')}{text}{_RESET}"
        return text


class FleetLogger(logging.Logger):
    """``logging.Logger`` with ``train``/``eval`` helpers."""

    def train(self, msg, *args, **kwargs):
        if self.isEnabledFor(TRAIN_LEVEL):
            self._log(TRAIN_LEVEL, msg, args, **kwargs)

    def eval(self, msg, *args, **kwargs):
        if self.isEnabledFor(EVAL_LEVEL):
            self._log(EVAL_LEVEL, msg, args, **kwargs)


def _build() -> FleetLogger:
    logging.setLoggerClass(FleetLogger)
    lg = logging.getLogger("paddlefleetx_b200")
    logging.setLoggerClass(logging.Logger)
    lg.propagate = False
    if not lg.handlers:
        handler = logging.StreamHandler(sys.stdout)
        use_color = sys.stdout.isatty() or os.environ.get("PFX_FORCE_COLOR") == "1"
        handler.setFormatter(_AnsiFormatter(use_color))
        lg.addHandler(handler)
    lg.setLevel(os.environ.get("PFX_LOG_LEVEL", "INFO"))
    return lg  # type: ignore[return-value]


logger: FleetLogger = _build()


class Logger:
    """Object-style logger of the reference (utils/log.py:65-150): ``log.info(msg)`` / ``log.TRAIN(msg)`` / ``log(level, msg)``, a global
    ``disable()`` / ``enable()`` switch, ``use_terminator`` to rewrite one console line, and ``processing(msg)`` — a spinner that runs while
    the ``with`` body works.  Records go through the same handler / formatter as the module-level ``logger``."""

    LEVELS = {"DEBUG": logging.DEBUG, "INFO": logging.INFO, "TRAIN": TRAIN_LEVEL, "EVAL": EVAL_LEVEL, "WARNING": logging.WARNING,
              "ERROR": logging.ERROR, "CRITICAL": logging.CRITICAL}

    def __init__(self, name: str = None):
        self.logger = logging.getLogger(name or "PaddleFleetX")
        self.handler = logging.StreamHandler(sys.stdout)
        self.handler.setFormatter(_AnsiFormatter(sys.stdout.isatty() or os.environ.get("PFX_FORCE_COLOR") == "1"))
        if not self.logger.handlers:
            self.logger.addHandler(self.handler)
        else:
            self.handler = self.logger.handlers[0]
        self.logLevel = "DEBUG"
        self.logger.setLevel(logging.DEBUG)
        self.logger.propagate = False
        self._is_enable = True
        for key, level in self.LEVELS.items():

            def emit(msg, _level=level):
                self(_level, msg)

            self.__dict__[key] = emit
            self.__dict__[key.lower()] = emit

    def disable(self):
        self._is_enable = False

    def enable(self):
        self._is_enable = True

    @property
    def is_enable(self) -> bool:
        return self._is_enable

    def __call__(self, log_level, msg: str):
        if self._is_enable:
            self.logger.log(self.LEVELS.get(log_level, log_level) if isinstance(log_level, str) else log_level, msg)

    @contextlib.contextmanager
    def use_terminator(self, terminator: str):
        old, self.handler.terminator = self.handler.terminator, terminator
        try:
            yield
        finally:
            self.handler.terminator = old

    @contextlib.contextmanager
    def processing(self, msg: str, interval: float = 0.1):
        stop = threading.Event()

        def spin():
            i = 0
            while not stop.is_set():
                with self.use_terminator("\r"):
                    self.info(f"{msg}: {'\\|/-'[i % 4]}")
                stop.wait(interval)
                i += 1

        t = threading.Thread(target=spin, daemon=True)
        t.start()
        try:
            yield
        finally:
            stop.set()
            t.join()


def advertise() -> None:
    """Banner shown above the config dump (reference: utils/log.py advertise())."""
    title = "PaddleFleetX-H100"
    sub = "Hopper-native (H100) large-model training suite"
    width = max(len(title), len(sub)) + 8
    bar = "=" * width
    logger.info(bar)
    logger.info(title.center(width))
    logger.info(sub.center(width))
    logger.info(bar)


def device_synchronize() -> None:
    import torch

    if torch.cuda.is_available():
        torch.cuda.synchronize()


def convert_timestamp_to_data(timeStamp) -> str:
    """Seconds -> ``H:MM:SS`` (the ETA field of the train line; reference utils/log.py:188-189)."""
    return str(datetime.timedelta(seconds=int(timeStamp)))


def get_timestamp() -> float:
    """Wall-clock after a device sync (reference: utils/log.py:180-186)."""
    device_synchronize()
    return time.time()
