"""TEST INFRASTRUCTURE: start the ranks of a torch.distributed group as processes on this host and collect their output."""
import os
import subprocess
import sys
import zlib


def run_ranks(world, argv_or_code, salt, timeout=300):
    """Run ``world`` Python processes with RANK / WORLD_SIZE / MASTER_ADDR / MASTER_PORT set: ``python *argv`` for a
    list, ``python -c code`` for a string.  The port depends on this process's pid, ``world`` and ``salt``; every caller
    passes its own salt (including whatever its parameters are), so tests running side by side pick different ports.
    -> [(returncode, stdout and stderr)] in rank order.  A rank still running when one times out is killed."""
    port = 20000 + (os.getpid() * 7 + world * 13 + zlib.crc32(salt.encode())) % 12000
    cmd = [sys.executable, "-c", argv_or_code] if isinstance(argv_or_code, str) else [sys.executable, *argv_or_code]
    procs = []
    try:
        for r in range(world):
            env = dict(os.environ, RANK=str(r), WORLD_SIZE=str(world), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
            procs.append(subprocess.Popen(cmd, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True))
        outs = []
        for p in procs:
            out, _ = p.communicate(timeout=timeout)
            outs.append((p.returncode, out))
        return outs
    finally:
        for p in procs:
            if p.poll() is None:
                p.kill()
                p.wait()
