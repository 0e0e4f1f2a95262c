"""Host watchdog: the reference inherits NCCL's watchdog/heartbeat threads; ours is a
small thread that (a) publishes a heartbeat key in the store, (b) notices peers whose heartbeat
stops and (c) aborts this process with a diagnostic (flight-recorder dump) instead of letting a
device-side spin-wait hang forever.  Device-side waits additionally carry their own
``globaltimer`` timeout (csrc/cuda/symm_kernels.cu)."""
from __future__ import annotations

import os
import sys
import threading
import time
from typing import Optional


class Watchdog:
    def __init__(self, group=None, interval: float = 1.0, timeout: float = 60.0, abort: bool = True):
        from .. import distributed as dist

        self.group = group or dist.get_default_group()
        self.interval, self.timeout, self.abort = interval, timeout, abort
        self._stop = threading.Event()
        self._thread: Optional[threading.Thread] = None
        self.dead_peers = []

    def _key(self, r):
        return f"watchdog/hb/{r}"

    def start(self):
        self._thread = threading.Thread(target=self._run, name="pdt-watchdog", daemon=True)
        self._thread.start()
        return self

    def stop(self):
        self._stop.set()
        if self._thread is not None:
            self._thread.join(self.interval * 2 + 1)

    def _run(self):
        g = self.group
        last_seen = {r: (time.time(), None) for r in range(g.size())}
        while not self._stop.wait(self.interval):
            now = time.time()
            try:
                g.store.set(self._key(g.rank()), str(now))
                for r in range(g.size()):
                    if r == g.rank() or not g.store.check([self._key(r)]):
                        continue
                    v = g.store.get(self._key(r))
                    if v != last_seen[r][1]:
                        last_seen[r] = (now, v)
            except Exception:  # store gone: rank 0 died
                self.dead_peers = [0]
                break
            self.dead_peers = [r for r, (t, v) in last_seen.items()
                               if r != g.rank() and v is not None and now - t > self.timeout]
            if self.dead_peers:
                break
        if self.dead_peers and not self._stop.is_set():
            sys.stderr.write(f"[rank{g.rank()}] watchdog: no heartbeat from ranks {self.dead_peers} for "
                             f"{self.timeout}s; recent collectives: {g.comm.flight_records()[-8:]}\n")
            sys.stderr.flush()
            if self.abort:
                os._exit(86)
