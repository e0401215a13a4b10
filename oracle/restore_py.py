"""oracle/restore_py.py — CPU restatement of placement-state restore (include/egpu_restore.h).

TEST INFRASTRUCTURE ONLY: imported by tests/ and scripts that generate golden vectors; never
by the product package.

What is pinned to the reference (elastic-ai/elastic-gpu-agent @ 2609107) and what is not:
  PINNED    the stored formats — record key "namespace/name" and value
            json.Marshal(map[container]*Device) (pkg/types/pod.go:39-58, Device fields
            pkg/types/device.go:11-15), symlink "elastic-gpu-<Hash>-<i>" -> "/dev/nvidia<N>"
            (pkg/operator/gpushare.go:10-14,31-55) — and the identity check
            Hash == hex(sha256(":".join(sorted(List))))[:8] (pkg/types/device.go:17-25,49-54),
            here through Python's json and hashlib.
  UNPINNED  the restore rule itself: GPUManager.Restore() is declared and never implemented
            (pkg/manager/manager.go:20).  It follows DESIGN.md §2.7 with the units the reference
            uses when it creates the links: len(List) percent for gpu-core, len(List)/100 whole
            cards above 100 (pkg/plugins/gpushare.go:62-69,127-128; base.go:282-292), len(List)
            MiB for gpu-memory (pkg/plugins/gpushare.go:159-168).
"""
from __future__ import annotations

import hashlib
import json
import re

REC_OK, REC_EMPTY, REC_FOREIGN, REC_NO_LINK, REC_HASH_MISMATCH = range(5)
CORE = "elasticgpu.io/gpu-core"
MEM = "elasticgpu.io/gpu-memory"

_LINK = re.compile(r"^(?:elastic-gpu-)?(.+)-(\d{1,9})$")
_TARGET = re.compile(r"^/dev/nvidia(\d{1,6})$")
_ID = re.compile(r"^[-0-9]{1,16}$")


class RestoreParseError(ValueError):
    pass


def device_hash(ids) -> str:
    return hashlib.sha256(":".join(sorted(ids)).encode()).hexdigest()[:8]


def _field(obj: dict, name: str):
    """encoding/json matches struct fields case-insensitively; the last duplicate wins."""
    out = None
    for k, v in obj.items():
        if k.lower() == name.lower():
            out = v
    return out


def parse_links(links) -> dict:
    table = {}
    for name, target in links:
        name = name.decode() if isinstance(name, bytes) else name
        target = target.decode() if isinstance(target, bytes) else target
        if name.startswith("elastic-gpuctl-"):
            continue
        m, t = _LINK.match(name), _TARGET.match(target)
        if not m or not t or int(m.group(2)) > 4096:
            continue
        table.setdefault(m.group(1), {})[int(m.group(2))] = int(t.group(1))
    return table


def restore(records, links, cap_core, cap_mem, verify: bool = True):
    """Returns (free_core, free_mem, oversub, counts[5], record_status)."""
    D = len(cap_core)
    link = parse_links(links)
    use_c = [0] * D
    use_m = [0] * D
    counts = [0] * 5
    rstat = []
    for r, (key, val) in enumerate(records):
        key = bytes(key)
        if key.count(b"/") != 1:
            raise RestoreParseError(f"error key format (record {r})")
        try:
            obj = json.loads(bytes(val).decode("utf-8", errors="replace"))
        except Exception as e:
            raise RestoreParseError(f"error val format (record {r})") from e
        if obj is None:
            obj = {}
        if not isinstance(obj, dict):
            raise RestoreParseError(f"error val format (record {r})")
        worst = REC_OK
        for _container, dev in obj.items():
            if dev is not None and not isinstance(dev, dict):
                raise RestoreParseError(f"error val format (record {r})")
            is_null = dev is None
            dev = dev or {}
            ids = _field(dev, "List") or []
            h = _field(dev, "Hash") or ""
            res = _field(dev, "ResourceName") or ""
            # json.Unmarshal into {Hash string; List []string; ResourceName string} rejects other types
            if not isinstance(h, str) or not isinstance(res, str) or not isinstance(ids, list) or \
                    any(not isinstance(i, str) for i in ids):
                raise RestoreParseError(f"error val format (record {r})")
            n = len(ids)
            if not is_null and res in (CORE, MEM):
                # IDs this plugin cannot have advertised ("%d-%02d", pkg/plugins/gpushare.go:28,163)
                if any(not _ID.match(i) for i in ids):
                    raise RestoreParseError(f"device ID is not \"<gpu>-<unit>\" (record {r})")
            if not is_null and res not in (CORE, MEM):
                st = REC_FOREIGN
            elif n == 0:
                st = REC_EMPTY
            elif verify and device_hash(ids) != h:
                st = REC_HASH_MISMATCH
            else:
                need = n // 100 if (res == CORE and n > 100) else 1
                gpus = [link.get(h, {}).get(i, -1) for i in range(need)]
                if any(g < 0 or g >= D for g in gpus):
                    st = REC_NO_LINK
                else:
                    st = REC_OK
                    if res == MEM:
                        use_m[gpus[0]] += n
                    elif n <= 100:
                        use_c[gpus[0]] += n
                    else:
                        for g in gpus:
                            use_c[g] += 100
            counts[st] += 1
            worst = max(worst, st)
        rstat.append(worst)
    free_c = [max(0, int(cap_core[d]) - use_c[d]) for d in range(D)]
    free_m = [max(0, int(cap_mem[d]) - use_m[d]) for d in range(D)]
    over = [int(int(cap_core[d]) < use_c[d] or int(cap_mem[d]) < use_m[d]) for d in range(D)]
    return free_c, free_m, over, counts, rstat


# ---- EGPU_RESTORE_CHARGE / EGPU_RESTORE_RELEASE: a few records applied to a live table -----------------
BIG = 1 << 40


class Refused(Exception):
    """EGPU_RESTORE_RELEASE refused (EGPU_ERR_STATE); args[0] is the first offending device"""


def usage(records, links, D, verify=True):
    """(use_core[D], use_mem[D], counts[5], record_status) of the records, by the restore rule: what a
    restore against an unbounded capacity takes away"""
    fc, fm, _, counts, rstat = restore(records, links, [BIG] * D, [BIG] * D, verify=verify)
    return [BIG - x for x in fc], [BIG - x for x in fm], counts, rstat


def charge(table, records, links, verify=True):
    """table = (free_core, free_mem, oversub): free' = max(free - U, 0), oversub' = oversub | (free - U < 0).
    Returns (table', counts, record_status)."""
    fc, fm, ov = table
    uc, um, counts, rstat = usage(records, links, len(fc), verify)
    c = [f - u for f, u in zip(fc, uc)]
    m = [f - u for f, u in zip(fm, um)]
    return ([max(x, 0) for x in c], [max(x, 0) for x in m],
            [int(bool(o) or x < 0 or y < 0) for o, x, y in zip(ov, c, m)]), counts, rstat


def release(table, records, links, cap_core, cap_mem, verify=True):
    """free' = free + U, flags unchanged, all or nothing: raises Refused on the first touched device that is
    oversubscribed or would exceed its capacity.  Returns (table', counts, record_status)."""
    fc, fm, ov = table
    uc, um, counts, rstat = usage(records, links, len(fc), verify)
    for d in range(len(fc)):
        if (uc[d] or um[d]) and (ov[d] or fc[d] + uc[d] > cap_core[d] or fm[d] + um[d] > cap_mem[d]):
            raise Refused(d)
    return ([f + u for f, u in zip(fc, uc)], [f + u for f, u in zip(fm, um)], list(ov)), counts, rstat


def marshal_record(namespace: str, name: str, containers: dict):
    """(key, value) as the reference writes them: PodInfo.Key() / Val() (pkg/types/pod.go:51-58).
    containers: {container: (ids, resource_name) | None}.  json.Marshal sorts map keys, writes the
    struct fields in declaration order (Hash, List, ResourceName) and no whitespace; NewDevice
    stores the list sorted."""
    parts = []
    for c in sorted(containers):
        d = containers[c]
        if d is None:
            parts.append(json.dumps(c) + ":null")
            continue
        ids, res = d
        ids = sorted(ids)
        body = ('{"Hash":' + json.dumps(device_hash(ids)) + ',"List":' + json.dumps(ids, separators=(",", ":")) +
                ',"ResourceName":' + json.dumps(res) + "}")
        parts.append(json.dumps(c) + ":" + body)
    return f"{namespace}/{name}".encode(), ("{" + ",".join(parts) + "}").encode()
