"""Distributed (sharded) checkpointing.

Reference parity (SURVEY D14, §3.5, §5.4): every worker writes ONLY its shards (flattened slices in the reference's
tensor-bundle format; plain tensor files + a JSON manifest here), directories `ckpt_<rank>_of_<n>/`, `max_to_keep`
rotation with a persisted prefix queue, "lazy save" when requested before the first step, restore by global step
reading only the slices this rank needs.
"""
from __future__ import annotations

import json
import os
import shutil
from typing import Any, Dict, List, Optional

import torch


class CheckpointManager:
    COMMIT = "COMMITTED"     # written into step_<n>/ after all ranks' shards of that step are on disk

    def __init__(self, root: str, rank: int, world: int, max_to_keep: int = 5):
        self.dir = os.path.join(root, f"ckpt_{rank}_of_{world}")
        self.rank, self.world, self.max_to_keep = rank, world, max_to_keep
        os.makedirs(self.dir, exist_ok=True)
        self.queue_file = os.path.join(self.dir, "checkpoint_queue.json")
        self.queue: List[int] = json.load(open(self.queue_file)) if os.path.exists(self.queue_file) else []
        self.lazy_request: Optional[int] = None

    # ------------------------------------------------------------------ save
    def request_save(self, global_step: int, warmed_up: bool) -> bool:
        """Returns True if the save can happen now; before the first step it is deferred (lazy save)."""
        if not warmed_up:
            self.lazy_request = global_step
            return False
        return True

    def save(self, executor, global_step: int, extra: Optional[Dict[str, Any]] = None) -> str:
        if hasattr(executor, "materialize_full_state"):
            executor.materialize_full_state()      # sharded-optimizer runs: make master / m / v whole before writing
        st = executor.store
        g = executor.g
        prefix = os.path.join(self.dir, f"step_{global_step}")
        tmp = prefix + ".tmp"
        os.makedirs(tmp, exist_ok=True)
        manifest: Dict[str, Any] = {"global_step": global_step, "rank": self.rank, "world": self.world, "vars": {},
                                    "step_count": executor.step_count, "drop_seed": executor.drop_seed, "extra": extra or {}}
        tensors: Dict[str, torch.Tensor] = {}
        # variables whose first / second moments live in the flat m / v buffers (others keep them as separate slot tensors)
        flat_moments = {pid for pid in st.order if st.moments_flat(pid)} if hasattr(st, "moments_flat") else set()
        for pid in st.order:
            n = g.nodes[pid]
            name = st.names[pid]
            tensors[name] = st.master_view(pid).detach().cpu().reshape(-1).clone()     # flattened shard, as the reference
            manifest["vars"][name] = {
                "shard_shape": list(st.shape[pid]), "full_shape": list(n.attrs.get("full_shape", st.shape[pid])),
                "shard_dims": list(n.attrs.get("shard_dims", [])), "shard_nums": list(n.attrs.get("shard_nums", [])),
                "shard_levels": list(n.attrs.get("shard_levels", [])), "coords": {str(k): v for k, v in executor.coords.items()},
                "flat_moments": pid in flat_moments,     # <name>/m, <name>/v below have the variable's shard shape
            }
            if pid in flat_moments:
                tensors[name + "/m"] = st._view(st.m, pid).detach().cpu().reshape(-1).clone()
                tensors[name + "/v"] = st._view(st.v, pid).detach().cpu().reshape(-1).clone()
        # optimizer slots outside the flat m / v buffers (momentum, Adafactor row / column statistics, SM3 accumulators,
        # separately stored shards of m / v): same shard description as a variable, under their own name
        manifest["slots"] = {}
        for n in getattr(st, "_state_nodes", []):
            if st.slot_is_live(n):
                t = st.state[n.id]
                tensors[n.name] = t.detach().cpu().reshape(-1).clone()
                manifest["slots"][n.name] = {
                    "shard_shape": list(t.shape), "full_shape": list(n.attrs.get("full_shape", t.shape)),
                    "shard_dims": list(n.attrs.get("shard_dims", [])), "shard_nums": list(n.attrs.get("shard_nums", [])),
                    "shard_levels": list(n.attrs.get("shard_levels", [])), "coords": {str(k): v for k, v in executor.coords.items()},
                }
        torch.save(tensors, os.path.join(tmp, "shards.pt"))
        json.dump(manifest, open(os.path.join(tmp, "manifest.json"), "w"))
        if os.path.exists(prefix):
            shutil.rmtree(prefix)
        os.replace(tmp, prefix)     # atomic publish of THIS rank's shards
        # commit: the step counts only once EVERY rank has published its shards -- a rank that died mid-save must not leave a
        # checkpoint that looks complete from the others' point of view (restore / latest() skip steps without the marker)
        import torch.distributed as dist
        if self.world > 1 and dist.is_available() and dist.is_initialized() and dist.get_world_size() == self.world:
            dist.barrier()
        open(os.path.join(prefix, self.COMMIT), "w").write(str(global_step))
        if global_step in self.queue:          # re-saving a step (lazy save then explicit save, resume then save) must not
            self.queue.remove(global_step)     # make rotation delete the directory that was just written
        self.queue.append(global_step)
        while len(self.queue) > self.max_to_keep:
            old = self.queue.pop(0)
            if old not in self.queue:
                shutil.rmtree(os.path.join(self.dir, f"step_{old}"), ignore_errors=True)
        json.dump(self.queue, open(self.queue_file, "w"))
        self.lazy_request = None
        return prefix

    def maybe_lazy_save(self, executor) -> Optional[str]:
        if self.lazy_request is not None:
            return self.save(executor, self.lazy_request)
        return None

    # ------------------------------------------------------------------ restore
    def committed(self, step: int, rank_dir: Optional[str] = None) -> bool:
        return os.path.exists(os.path.join(rank_dir or self.dir, f"step_{step}", self.COMMIT))

    def latest(self) -> Optional[int]:
        """Newest step of this rank's queue whose save completed on every rank."""
        for step in reversed(self.queue):
            if self.committed(step):
                return step
        return None

    def restore(self, executor, global_step: Optional[int] = None) -> int:
        step = self.latest() if global_step is None else global_step
        if step is None:
            step = self._latest_any_layout()
        if step is None:
            raise FileNotFoundError("no checkpoint to restore")
        prefix = os.path.join(self.dir, f"step_{step}")
        st = executor.store
        if os.path.isdir(prefix) and not self.committed(step):
            raise FileNotFoundError(f"checkpoint step {step} was never committed (a rank failed while saving it)")
        same_layout = os.path.exists(os.path.join(prefix, "manifest.json"))
        if same_layout:
            manifest = json.load(open(os.path.join(prefix, "manifest.json")))
            same_layout = all(tuple(manifest["vars"].get(st.names[pid], {}).get("shard_shape", ())) == tuple(st.shape[pid])
                              and manifest["vars"][st.names[pid]].get("coords") == {str(k): v for k, v in executor.coords.items()}
                              for pid in st.order)
        if not same_layout:
            return self._restore_resharded(executor, step)
        tensors = torch.load(os.path.join(prefix, "shards.pt"))
        for pid in st.order:
            name = st.names[pid]
            st.master_view(pid).copy_(tensors[name].reshape(st.shape[pid]).to(st.device))
            if st.m is not None and name + "/m" in tensors and manifest["vars"][name].get("flat_moments", True):
                st._view(st.m, pid).copy_(tensors[name + "/m"].reshape(st.shape[pid]).to(st.device))
                st._view(st.v, pid).copy_(tensors[name + "/v"].reshape(st.shape[pid]).to(st.device))
        for n in getattr(st, "_state_nodes", []):
            if n.name in manifest.get("slots", {}) and n.name in tensors and st.slot_is_live(n):
                st.state[n.id].copy_(tensors[n.name].reshape(st.state[n.id].shape).to(st.device))
        st.sync_compute()
        executor.step_count = int(manifest.get("step_count", step))
        executor.drop_seed = int(manifest.get("drop_seed", executor.drop_seed))   # a resumed run drops what the first would have
        return step

    # ------------------------------------------------------------------ restore into a DIFFERENT plan / world size
    def _all_rank_dirs(self) -> List[str]:
        root = os.path.dirname(self.dir)
        return sorted(os.path.join(root, d) for d in os.listdir(root) if d.startswith("ckpt_") and "_of_" in d)

    def _latest_any_layout(self) -> Optional[int]:
        best = None
        for d in self._all_rank_dirs():
            qf = os.path.join(d, "checkpoint_queue.json")
            if os.path.exists(qf):
                q = [s_ for s_ in json.load(open(qf)) if self.committed(s_, d)]
                if q:
                    best = q[-1] if best is None else max(best, q[-1])
        return best

    def _restore_resharded(self, executor, step: int) -> int:
        """The checkpoint was written by a different plan (other world size / sharding): rebuild every variable from the
        shards of ALL writer ranks (each shard is placed by its recorded shard_dims / nums / levels / coords), then cut out
        what THIS rank's plan stores.  Needs the writers' directories on a shared filesystem (one box: always true)."""
        writers = []
        for d in self._all_rank_dirs():
            pf = os.path.join(d, f"step_{step}")
            if os.path.exists(os.path.join(pf, "manifest.json")):
                writers.append((json.load(open(os.path.join(pf, "manifest.json"))), torch.load(os.path.join(pf, "shards.pt"))))
        if not writers:
            raise FileNotFoundError(f"no shards of step {step} under {os.path.dirname(self.dir)}")
        world_w = writers[0][0]["world"]
        writers = [w for w in writers if w[0]["world"] == world_w]
        if len(writers) != world_w:
            raise FileNotFoundError(f"step {step}: found {len(writers)} of {world_w} writer shards")
        st, g = executor.store, executor.g

        def assemble(name: str, suffix: str, section: str = "vars") -> Optional[torch.Tensor]:
            full = None
            for man, tens in writers:
                meta = man.get(section, {}).get(name)
                if meta is None or name + suffix not in tens:
                    continue         # (a pipeline writer holds only its own stage's variables)
                if suffix and not meta.get("flat_moments", True):
                    return None      # (the writer kept its moments as separately sharded slots: see the "slots" section)
                if full is None:
                    full = torch.zeros(meta["full_shape"], dtype=torch.float32)
                    covered = torch.zeros(meta["full_shape"], dtype=torch.bool)
                view, cview = full, covered
                for d_, n_, l_ in zip(meta["shard_dims"], meta["shard_nums"], meta["shard_levels"]):
                    sz = view.shape[d_] // n_
                    o_ = int(meta["coords"].get(str(l_), 0)) * sz
                    view, cview = view.narrow(d_, o_, sz), cview.narrow(d_, o_, sz)
                view.copy_(tens[name + suffix].reshape(meta["shard_shape"]))
                cview.fill_(True)
            if full is not None and not bool(covered.all()):
                raise FileNotFoundError(f"checkpoint step {step}: the shards found for {name + suffix} do not cover the whole tensor")
            return full

        from ..runtime.executor import shard_of
        for pid in st.order:
            name = st.names[pid]
            attrs = g.nodes[pid].attrs
            for suffix, dst in (("", st.master_view(pid)), ("/m", None if st.m is None else st._view(st.m, pid)),
                                ("/v", None if st.v is None else st._view(st.v, pid))):
                if dst is None:
                    continue
                full = assemble(name, suffix)
                if full is None and suffix:
                    full = assemble(name + suffix, "", "slots")      # the writer kept this moment as a separately sharded slot
                if full is None:
                    if suffix == "":
                        raise KeyError(f"variable {name} missing from checkpoint step {step}")
                    continue
                dst.copy_(shard_of(full, attrs, executor.coords).reshape(dst.shape).to(st.device))
        # optimizer slots by name.  Writer and reader may disagree on WHERE a moment lives (flat m / v buffers vs a separately
        # sharded slot tensor, e.g. LAMB under a ZeRO plan vs one process), so every reader slot looks in the writers' "slots"
        # section first and, for <var>/m and <var>/v, in the variable section second.
        if hasattr(st, "ensure_slots"):
            st.ensure_slots()
        for n in getattr(st, "_state_nodes", []):
            if n.id not in st.state:
                continue
            full = assemble(n.name, "", "slots")
            if full is None and (n.name.endswith("/m") or n.name.endswith("/v")):
                full = assemble(n.name[:-2], n.name[-2:])
            if full is not None:
                st.state[n.id].copy_(shard_of(full, n.attrs, executor.coords).reshape(st.state[n.id].shape).to(st.device))
        st.sync_compute()
        executor.step_count = int(writers[0][0].get("step_count", step))
        executor.drop_seed = int(writers[0][0].get("drop_seed", executor.drop_seed))
        return step
