#!/usr/bin/env python
"""Fake `zfs` for plumbing tests and the CPU plumbing baseline (SURVEY.md 4, 8d
config 1): selected through the reference's own `zfsPath` knob
(lib/backupSender.js:177, lib/zfsClient.js:793) and put first on PATH for the bare
`zfs list` of lib/backupSender.js:253.

  zfs list -t snapshot -H -d 1 -S name -o name <ds>   -> <ds>@<13 digits> lines
  zfs send -v -P <snap>    -> stream from $FAKE_ZFS_STREAM on stdout, the
                              `full/size/HH:MM:SS` progress protocol on stderr
  zfs send -c -v -P <snap> -> the same, from $FAKE_ZFS_STREAM_C when it is set
                              ($FAKE_ZFS_SEND_ARGS: every send appends its arguments, one JSON list a line)
  zfs recv -v -u <ds>      -> drains stdin, writes sha256 + byte count to $FAKE_ZFS_RECV_OUT

With $FAKE_ZFS_STATE (a JSON file, flock-protected) it also keeps a tiny pool model
for the dataset lifecycle either side of the path (SURVEY.md 8f f3/f4):
  list -Hp -o name | set | get -Hp | inherit | rename [-p] | mount | unmount |
  snapshot | destroy [-r] | create [-o k=v]
  state = {"datasets": {name: {"props": {}, "mounted": bool, "busy": bool,
                               "snapshots": [[name, creation], ...]}},
           "held": [snapshot, ...], "clock": n}
  * `send` holds its snapshot while it streams (a snapshot being sent cannot be
    destroyed: `destroy` fails with "dataset is busy"), `recv` creates the dataset
    unmounted (-u) with the sent snapshot.
"""
import contextlib
import fcntl
import hashlib
import json
import os
import sys
import time


@contextlib.contextmanager
def state(write=True):
    path = os.environ["FAKE_ZFS_STATE"]
    with open(path, "a+") as f:
        fcntl.flock(f, fcntl.LOCK_EX)
        f.seek(0)
        raw = f.read()
        st = json.loads(raw) if raw.strip() else {}
        st.setdefault("datasets", {})
        st.setdefault("held", [])
        st.setdefault("clock", 0)
        yield st
        if write:
            f.seek(0)
            f.truncate()
            f.write(json.dumps(st))
            f.flush()


def die(msg, rc=1):
    sys.stderr.write("cannot %s\n" % msg)
    return rc


def new_ds():
    return {"props": {}, "mounted": False, "busy": False, "snapshots": []}


def meta(a):
    """dataset lifecycle commands against the state file"""
    cmd = a[0]
    with state() as st:
        ds = st["datasets"]
        if cmd == "list" and "-t" not in a:
            sys.stdout.write("".join(n + "\n" for n in sorted(ds)))
            return 0
        if cmd == "list":
            name = a[-1]
            if name not in ds:
                return die("open '%s': dataset does not exist" % name)
            snaps = list(ds[name]["snapshots"])
            if "-S" in a:                                    # descending by name (sender)
                snaps.sort(key=lambda s: s[0], reverse=True)
            else:                                            # -s creation: oldest first (snapshotter)
                snaps.sort(key=lambda s: s[1])
            sys.stdout.write("".join("%s@%s\n" % (name, s[0]) for s in snaps))
            return 0
        if cmd == "set":
            kv, name = a[1], a[2]
            if name not in ds:
                return die("open '%s': dataset does not exist" % name)
            k, v = kv.split("=", 1)
            if k == "canmount" and v == "off" and ds[name]["mounted"]:
                if ds[name]["busy"]:
                    return die("unmount '%s': Device busy" % name)
                ds[name]["mounted"] = False
            ds[name]["props"][k] = v
            return 0
        if cmd == "get":
            prop, name = a[-2], a[-1]
            if name not in ds:
                return die("open '%s': dataset does not exist" % name)
            if prop == "mounted":
                val, src = ("yes" if ds[name]["mounted"] else "no"), "-"
            elif prop in ds[name]["props"]:
                val, src = ds[name]["props"][prop], "local"
            else:
                val, src = "-", "default"
            sys.stdout.write("%s\t%s\t%s\t%s\n" % (name, prop, val, src))
            return 0
        if cmd == "inherit":
            prop, name = a[1], a[2]
            if name not in ds:
                return die("open '%s': dataset does not exist" % name)
            ds[name]["props"].pop(prop, None)
            return 0
        if cmd == "rename":
            parents = "-p" in a
            src, dst = a[-2], a[-1]
            if src not in ds:
                return die("open '%s': dataset does not exist" % src)
            if dst in ds:
                return die("rename to '%s': dataset already exists" % dst)
            parent = os.path.dirname(dst)
            if parent and parent not in ds:
                if not parents:
                    return die("rename to '%s': parent does not exist" % dst)
                p = parent
                while p and p not in ds and "/" in p:
                    ds[p] = new_ds()
                    p = os.path.dirname(p)
            for n in [n for n in ds if n == src or n.startswith(src + "/")]:
                ds[dst + n[len(src):]] = ds.pop(n)
            st["held"] = [dst + h[len(src):] if (h.startswith(src + "@") or h.startswith(src + "/")) else h
                          for h in st["held"]]
            return 0
        if cmd == "mount":
            name = a[-1]
            if name not in ds:
                return die("open '%s': dataset does not exist" % name)
            if ds[name]["props"].get("canmount") == "off":
                return die("mount '%s': 'canmount' property is set to 'off'" % name)
            if ds[name]["mounted"]:
                return die("mount '%s': filesystem already mounted" % name)
            ds[name]["mounted"] = True
            return 0
        if cmd in ("unmount", "umount"):
            name = a[-1]
            if name not in ds:
                return die("open '%s': dataset does not exist" % name)
            if ds[name]["busy"] and "-f" not in a:
                return die("unmount '%s': Device busy" % name)
            ds[name]["mounted"] = False
            return 0
        if cmd == "snapshot":
            full = a[-1]
            name, _, snap = full.partition("@")
            if name not in ds:
                return die("open '%s': dataset does not exist" % name)
            if any(s[0] == snap for s in ds[name]["snapshots"]):
                return die("create snapshot '%s': dataset already exists" % full)
            st["clock"] += 1
            ds[name]["snapshots"].append([snap, st["clock"]])
            return 0
        if cmd == "destroy":
            target = a[-1]
            if "@" in target:
                name, _, snap = target.partition("@")
                if name not in ds or not any(s[0] == snap for s in ds[name]["snapshots"]):
                    return die("open '%s': dataset does not exist" % target)
                if target in st["held"]:
                    return die("destroy '%s': dataset is busy" % target)
                ds[name]["snapshots"] = [s for s in ds[name]["snapshots"] if s[0] != snap]
                return 0
            if target not in ds:
                return die("open '%s': dataset does not exist" % target)
            kids = [n for n in ds if n.startswith(target + "/")]
            if (kids or ds[target]["snapshots"]) and "-r" not in a:
                return die("destroy '%s': filesystem has children" % target)
            for n in kids + [target]:
                ds.pop(n)
            return 0
        if cmd == "create":
            name = a[-1]
            if name in ds:
                return die("create '%s': dataset already exists" % name)
            d = new_ds()
            i = 1
            while i < len(a) - 1:
                if a[i] == "-o":
                    k, v = a[i + 1].split("=", 1)
                    d["props"][k] = v
                    i += 2
                else:
                    i += 1
            d["mounted"] = d["props"].get("canmount", "on") == "on"
            ds[name] = d
            return 0
    return die("%s: unsupported by fake zfs" % cmd, 2)


def main():
    a = sys.argv[1:]
    if not a:
        return 2
    stateful = bool(os.environ.get("FAKE_ZFS_STATE"))
    if a[0] == "list":
        if "-t" not in a:
            return meta(a) if stateful else 0
        ds = a[-1]
        if stateful:
            with state(write=False) as st:
                known = ds in st["datasets"]
            if known:                                        # modelled dataset: list from the pool model
                return meta(a)
        if os.environ.get("FAKE_ZFS_NO_SNAPSHOTS"):
            return 0
        sys.stdout.write("%s@operator-made\n%s@1405378955344\n%s@1405378000000\n" % (ds, ds, ds))
        return 0
    if a[0] == "send":
        snap = a[-1]
        if os.environ.get("FAKE_ZFS_SEND_COUNT"):
            with open(os.environ["FAKE_ZFS_SEND_COUNT"], "a") as f:
                f.write("send\n")
        if stateful:
            with state() as st:
                st["held"].append(snap)
        if os.environ.get("FAKE_ZFS_SEND_ARGS"):
            with open(os.environ["FAKE_ZFS_SEND_ARGS"], "a") as f:
                f.write(json.dumps(a) + "\n")
        try:
            path = os.environ["FAKE_ZFS_STREAM"]
            if "-c" in a[1:-1] and os.environ.get("FAKE_ZFS_STREAM_C"):
                path = os.environ["FAKE_ZFS_STREAM_C"]
            size = os.path.getsize(path)
            sys.stderr.write("full\t%s\t%d\nsize\t%d\n" % (snap, size, size))
            sys.stderr.flush()
            sent = 0
            fail_at = int(os.environ.get("FAKE_ZFS_SEND_FAIL_AT", "-1"))
            delay = float(os.environ.get("FAKE_ZFS_SEND_DELAY", "0"))
            out = sys.stdout.buffer
            with open(path, "rb") as f:
                while True:
                    buf = f.read(1 << 20)
                    if not buf:
                        break
                    out.write(buf)
                    sent += len(buf)
                    sys.stderr.write("%s\t%d\t%s\n" % (time.strftime("%H:%M:%S"), sent, snap))
                    sys.stderr.flush()
                    if delay:
                        out.flush()
                        time.sleep(delay)
                    if 0 <= fail_at <= sent:
                        sys.stderr.write("internal error: fake failure\n")
                        return 1
            out.flush()
            return 0
        finally:
            if stateful:
                with state() as st:
                    if snap in st["held"]:
                        st["held"].remove(snap)
    if a[0] in ("recv", "receive"):
        h = hashlib.sha256()
        n = 0
        inp = sys.stdin.buffer
        while True:
            buf = inp.read(1 << 20)
            if not buf:
                break
            h.update(buf)
            n += len(buf)
        with open(os.environ["FAKE_ZFS_RECV_OUT"], "w") as f:
            f.write("%s %d\n" % (h.hexdigest(), n))
        if stateful:
            with state() as st:
                name = a[-1]
                if name in st["datasets"]:
                    return die("receive into '%s': destination exists" % name)
                p = os.path.dirname(name)
                while p and p not in st["datasets"] and "/" in p:
                    st["datasets"][p] = new_ds()
                    p = os.path.dirname(p)
                d = new_ds()                                  # -u: not mounted
                st["clock"] += 1
                d["snapshots"].append([os.environ.get("FAKE_ZFS_RECV_SNAP", "1405378955344"), st["clock"]])
                st["datasets"][name] = d
        sys.stderr.write("received %d bytes\n" % n)
        return 0
    if stateful:
        return meta(a)
    return 0


if __name__ == "__main__":
    sys.exit(main())
