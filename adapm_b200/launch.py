"""Job launcher (the reference's ``tracker/dmlc_local.py`` / ``dmlc_mpi.py`` equivalent).

    python -m adapm_b200.launch -s N [--backend cpu|cuda] <script.py | -m module> [args...]

Starts N ranks on this host (one per GPU for ``--backend cuda``) with ``RANK / LOCAL_RANK /
WORLD_SIZE / MASTER_ADDR / MASTER_PORT / ADAPM_JOB`` (plus the reference's ``DMLC_NUM_SERVER /
DMLC_ROLE / DMLC_RANK / DMLC_PS_ROOT_URI / DMLC_PS_ROOT_PORT`` for scripts that read them) and no
scheduler process: ranks rendezvous through a POSIX-shm control block. A rank that exits with
code 254 is restarted (``keepalive`` of tracker/dmlc_local.py:15-26). ``torchrun`` and ``mpirun``
work too - the package also reads ``OMPI_COMM_WORLD_*``, ``PMI_*`` and ``SLURM_*``.
The fabric is single-node (shm control block + peer-mapped heaps over NVLink/NVSwitch): one 8-GPU NVSwitch box is the target.
"""
from __future__ import annotations

import argparse
import os
import shlex
import socket
import subprocess
import sys
import threading
import uuid


def _free_port() -> int:
    from .utils.net import get_available_port

    return get_available_port("127.0.0.1")


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(prog="adapm_b200.launch", description=__doc__,
                                 formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("-s", "--num-servers", type=int, required=True, help="number of ranks (= PS nodes = GPUs)")
    ap.add_argument("-n", "--num-workers", type=int, default=0, help="accepted for parity with dmlc_local.py (ignored)")
    ap.add_argument("--backend", default=None, choices=["cpu", "cuda"])
    ap.add_argument("--log-dir", default=None, help="write one log file per rank")
    ap.add_argument("--env", action="append", default=[], help="extra KEY=VALUE for every rank")
    ap.add_argument("--launcher", default="local", choices=["local", "mpi", "ssh"],
                    help="local: threads spawning the ranks here (dmlc_local.py); mpi: one mpirun (dmlc_mpi.py); "
                         "ssh: one ssh session per rank on the host of --hostfile (dmlc_ssh.py)")
    ap.add_argument("-H", "--hostfile", default=None, help="ssh launcher: file with the target host (one line)")
    ap.add_argument("--sync-dst-dir", default=None, help="ssh launcher: rsync the working directory there first")
    ap.add_argument("--dry-run", action="store_true", help="print the launch commands instead of running them")
    ap.add_argument("-m", dest="module", default=None, help="run a module instead of a script")
    ap.add_argument("command", nargs=argparse.REMAINDER)
    a = ap.parse_args(argv)
    if a.module is None and not a.command:
        ap.error("nothing to launch")
    cmd = [sys.executable] + (["-m", a.module] if a.module else []) + a.command
    port = _free_port()
    job = f"L{os.getpid()}_{uuid.uuid4().hex[:8]}"
    codes = [None] * a.num_servers
    common = {"WORLD_SIZE": str(a.num_servers), "MASTER_ADDR": "127.0.0.1", "MASTER_PORT": str(port), "ADAPM_JOB": job,
              "DMLC_NUM_SERVER": str(a.num_servers), "DMLC_NUM_WORKER": "0", "DMLC_ROLE": "server",
              "DMLC_PS_ROOT_URI": "127.0.0.1", "DMLC_PS_ROOT_PORT": str(port)}
    if a.backend:
        common["ADAPM_BACKEND"] = a.backend
    for kv in a.env:
        k, _, v = kv.partition("=")
        common[k] = v

    if a.launcher == "mpi":
        # one mpirun; the ranks read OMPI_COMM_WORLD_RANK / PMI_RANK (adapm_b200/__init__.py), env goes via -x
        mpi = ["mpirun", "-n", str(a.num_servers)] + (["--allow-run-as-root"] if os.geteuid() == 0 else [])
        for k, v in common.items():
            mpi += ["-x", f"{k}={v}"]
        mpi += cmd
        if a.dry_run:
            print(" ".join(shlex.quote(x) for x in mpi))
            return 0
        return subprocess.call(mpi)

    ssh_host = None
    if a.launcher == "ssh":
        hosts = [h.split()[0] for h in open(a.hostfile).read().splitlines() if h.strip() and not h.startswith("#")] \
            if a.hostfile else ["127.0.0.1"]
        if len(set(hosts)) != 1:
            print("[launch] the fabric is single-node (shm control block + peer-mapped heaps, NVSwitch): the hostfile must name exactly "
                  "one host; all ranks of a job share one box", file=sys.stderr)
            return 2
        ssh_host = hosts[0]
        if a.sync_dst_dir:
            rs = ["rsync", "-az", "--exclude", ".git", os.getcwd() + "/", f"{ssh_host}:{a.sync_dst_dir}/"]
            if a.dry_run:
                print(" ".join(shlex.quote(x) for x in rs))
            elif subprocess.call(rs) != 0:
                return 1

    def ssh_command(rank: int) -> list:
        envs = dict(common, RANK=str(rank), LOCAL_RANK=str(rank), DMLC_RANK=str(rank))
        wd = a.sync_dst_dir or os.getcwd()
        remote = "cd " + shlex.quote(wd) + " && env " + " ".join(f"{k}={shlex.quote(v)}" for k, v in envs.items()) \
                 + " " + " ".join(shlex.quote(x) for x in cmd)
        return ["ssh", "-o", "StrictHostKeyChecking=no", ssh_host, remote]

    if a.launcher == "ssh" and a.dry_run:
        for r in range(a.num_servers):
            print(" ".join(shlex.quote(x) for x in ssh_command(r)))
        return 0

    def run(rank: int) -> None:
        env = dict(os.environ)
        env.update({"RANK": str(rank), "LOCAL_RANK": str(rank), "WORLD_SIZE": str(a.num_servers),
                    "MASTER_ADDR": "127.0.0.1", "MASTER_PORT": str(port), "ADAPM_JOB": job,
                    "DMLC_NUM_SERVER": str(a.num_servers), "DMLC_NUM_WORKER": "0", "DMLC_ROLE": "server",
                    "DMLC_RANK": str(rank), "DMLC_PS_ROOT_URI": "127.0.0.1", "DMLC_PS_ROOT_PORT": str(port)})
        if a.backend:
            env["ADAPM_BACKEND"] = a.backend
        for kv in a.env:
            k, _, v = kv.partition("=")
            env[k] = v
        while True:
            out = open(os.path.join(a.log_dir, f"rank{rank}.log"), "ab") if a.log_dir else None
            rc = subprocess.call(ssh_command(rank) if ssh_host else cmd, env=env, stdout=out,
                                 stderr=subprocess.STDOUT if out else None)
            if out:
                out.close()
            if rc != 254:  # keepalive: restart on 254
                codes[rank] = rc
                return

    if a.log_dir:
        os.makedirs(a.log_dir, exist_ok=True)
    ths = [threading.Thread(target=run, args=(r,)) for r in range(a.num_servers)]
    [t.start() for t in ths]
    [t.join() for t in ths]
    bad = [(r, c) for r, c in enumerate(codes) if c != 0]
    if bad:
        print(f"[launch] ranks failed: {bad}", file=sys.stderr)
        return 1
    return 0


if __name__ == "__main__":
    sys.exit(main())
