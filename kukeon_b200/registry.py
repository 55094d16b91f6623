"""Pool registry: the on-disk record of which checkpoints are resident ("next" row f1 of SURVEY.md §8(f)).

kukeon re-derives every piece of daemon state after a restart from files under its run path plus live
observation (internal/controller/runner/refresh.go:522), and guards the run path with an instance file
(internal/instance/instance.go:141 VerifyOrWrite).  GPU pools are different in one respect: device memory dies
with the daemon process, so a restarted kukeond can never re-adopt a pool — it can only *invalidate* what the
previous instance left behind (staged ipc.handle / manifest.json files that agent containers may still have
bind-mounted) and reload on demand.  This module is that logic, host-side only:

* `<run_path>/.kukeon-gpupool.json` — written with tmp + fsync + rename (internal/metadata/metadata.go:105-140);
  carries the daemon `epoch` (boot id : pid : process start time) and one entry per resident model.
* `PoolRegistry.reconcile()` at daemon start — entries of another epoch are stale: their staged mount directories are
  removed and they are returned so the caller can mark the cells that referenced them for reload.
* `record()` / `forget()` — called next to modelhub.Load / the last release.
"""
from __future__ import annotations

import json
import os
import shutil
import tempfile
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence

FILE_NAME = ".kukeon-gpupool.json"
API_VERSION = "kukeon.gpupool/v1"


def daemon_epoch(pid: Optional[int] = None) -> str:
    """boot-id : pid : start-time — changes whenever the process that owns the CUDA allocations changes."""
    pid = os.getpid() if pid is None else pid
    try:
        boot = open("/proc/sys/kernel/random/boot_id").read().strip()
    except OSError:
        boot = "unknown-boot"
    try:
        start = open(f"/proc/{pid}/stat").read().rsplit(")", 1)[1].split()[19]  # field 22: starttime (clock ticks)
    except (OSError, IndexError):
        start = "0"
    return f"{boot}:{pid}:{start}"


def _atomic_write(path: str, data: bytes, mode: int = 0o640) -> None:
    d = os.path.dirname(path)
    os.makedirs(d, mode=0o750, exist_ok=True)
    fd, tmp = tempfile.mkstemp(prefix=".kukeon-gpupool-", suffix=".tmp", dir=d)
    try:
        os.fchmod(fd, mode)
        os.write(fd, data)
        os.fsync(fd)
    finally:
        os.close(fd)
    os.rename(tmp, path)
    try:
        dfd = os.open(d, os.O_RDONLY)
        os.fsync(dfd)
        os.close(dfd)
    except OSError:
        pass


def shard_fingerprints(shards: List[str]) -> List[dict]:
    """Cheap identity of the files a pool was built from: (name, size, mtime_ns).  A changed fingerprint means the
    resident copy no longer matches the checkpoint on disk."""
    out = []
    for s in shards:
        st = os.stat(s)
        out.append({"file": s, "size": st.st_size, "mtime_ns": st.st_mtime_ns})
    return out


@dataclass
class Entry:
    key: str
    path: str
    mode: int
    file_bytes: int
    pool_bytes: int
    devices: List[int]
    shards: List[dict]
    mounts: List[str] = field(default_factory=list)  # staged <container>/gpupool directories
    # pipeline stage [begin, end) the pool holds; None: the whole checkpoint.  A restarted daemon reloads this stage, not the whole
    # model (which need not fit the devices).
    layers: Optional[List[int]] = None
    # PEFT LoRA adapter merged into the pool (kk_load_adapter); None: the base checkpoint alone.  A restarted daemon reloads base + adapter.
    adapter: Optional[str] = None

    def to_json(self) -> dict:
        d = dict(key=self.key, path=self.path, mode=self.mode, fileBytes=self.file_bytes, poolBytes=self.pool_bytes,
                 devices=self.devices, shards=self.shards, mounts=self.mounts)
        if self.layers is not None:
            d["layers"] = self.layers
        if self.adapter is not None:
            d["adapter"] = self.adapter
        return d

    @staticmethod
    def from_json(d: dict) -> "Entry":
        layers = d.get("layers")
        return Entry(d["key"], d["path"], d["mode"], d["fileBytes"], d["poolBytes"], list(d["devices"]), list(d["shards"]), list(d.get("mounts", [])),
                     None if layers is None else list(layers), d.get("adapter"))


class RegistryError(RuntimeError):
    pass


def _is_staged_dir(path: str) -> bool:
    """Directories Mount stages: <container>/gpupool (unnamed model) or <container>/gpupool/<name> (models[].name, validated to a single
    path component by schema.validate_models).  Anything else in a registry file is not ours to delete."""
    p = os.path.normpath(path)
    if os.path.basename(p) == "gpupool":
        return True
    parent = os.path.dirname(p)
    return os.path.basename(parent) == "gpupool" and os.path.basename(p) not in ("", ".", "..")


class PoolRegistry:
    def __init__(self, run_path: str, epoch: Optional[str] = None):
        self.run_path = run_path
        self.file = os.path.join(run_path, FILE_NAME)
        self.epoch = epoch or daemon_epoch()
        self.entries: Dict[str, Entry] = {}

    # -- persistence ---------------------------------------------------------------------------
    def _load(self):
        try:
            raw = open(self.file, "rb").read()
        except FileNotFoundError:
            return None
        try:
            doc = json.loads(raw)
            if doc.get("apiVersion") != API_VERSION or "epoch" not in doc:
                raise ValueError("unexpected document")
            return doc
        except (ValueError, KeyError) as e:
            raise RegistryError(f"parse {self.file}: {e}") from e

    def _save(self) -> None:
        doc = {"apiVersion": API_VERSION, "kind": "PoolRegistry", "epoch": self.epoch,
               "models": [e.to_json() for e in sorted(self.entries.values(), key=lambda e: e.key)]}
        _atomic_write(self.file, (json.dumps(doc, indent=2) + "\n").encode())

    # -- daemon start --------------------------------------------------------------------------
    def reconcile(self) -> List[Entry]:
        """Call once at daemon start.  Same epoch (e.g. a config reload in the same process): keep everything.
        Different epoch: every recorded pool died with its process — remove the staged mount directories, forget the
        entries and return them (the runner marks the cells that mounted them for reload)."""
        doc = self._load()
        if doc is None:
            self._save()
            return []
        prior = {e["key"]: Entry.from_json(e) for e in doc.get("models", [])}
        if doc["epoch"] == self.epoch:
            self.entries = prior
            return []
        stale = list(prior.values())
        for e in stale:
            for m in e.mounts:
                if _is_staged_dir(m):  # only ever delete directories we staged
                    shutil.rmtree(m, ignore_errors=True)
        self.entries = {}
        self._save()
        return stale

    # -- steady state --------------------------------------------------------------------------
    def record(self, key: str, path: str, mode: int, file_bytes: int, pool_bytes: int, devices: List[int], shards: List[str],
               mount_dir: Optional[str] = None, layers: Optional[Sequence[int]] = None, adapter: Optional[str] = None) -> Entry:
        e = self.entries.get(key)
        if e is None:
            e = Entry(key, path, mode, file_bytes, pool_bytes, sorted(devices), shard_fingerprints(shards),
                      layers=None if layers is None else list(layers), adapter=adapter)
            self.entries[key] = e
        if mount_dir and mount_dir not in e.mounts:
            e.mounts.append(mount_dir)
        self._save()
        return e

    def forget(self, key: str) -> None:
        if self.entries.pop(key, None) is not None:
            self._save()

    def drop_mount(self, key: str, mount_dir: str) -> None:
        e = self.entries.get(key)
        if e and mount_dir in e.mounts:
            e.mounts.remove(mount_dir)
            self._save()

    def changed_on_disk(self, key: str) -> bool:
        """True when a shard of a resident checkpoint was replaced since it was loaded (reload needed)."""
        e = self.entries[key]
        try:
            return shard_fingerprints([s["file"] for s in e.shards]) != e.shards
        except OSError:
            return True
