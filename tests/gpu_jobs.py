"""How the GPU tests run a job: one child process per GPU with the environment torchrun would give it."""
import os
import socket
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def run_ranks(script, args=(), nproc=1, env=None, timeout=600):
    """Run `python script *args` as ranks 0..nproc-1 (RANK, LOCAL_RANK, WORLD_SIZE, a rendezvous on a free port of
    127.0.0.1, the repository on PYTHONPATH, then `env`), print each rank's stdout and assert that every rank exited
    with 0.  On a timeout every rank is killed and the TimeoutExpired raised.  Returns [(returncode, stdout, stderr)]."""
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    procs = []
    for r in range(nproc):
        e = dict(os.environ, RANK=str(r), LOCAL_RANK=str(r), WORLD_SIZE=str(nproc), MASTER_ADDR="127.0.0.1",
                 MASTER_PORT=str(port), PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
        e.update(env or {})
        procs.append(subprocess.Popen([sys.executable, script, *args], env=e, stdout=subprocess.PIPE, stderr=subprocess.PIPE,
                                      text=True))
    outs = []
    for p in procs:
        try:
            o, err = p.communicate(timeout=timeout)
        except subprocess.TimeoutExpired:
            for q in procs:
                q.kill()
            raise
        outs.append((p.returncode, o, err))
    job = " ".join([os.path.relpath(script, ROOT), *args])
    for rc, o, err in outs:
        print(o)
        assert rc == 0, f"job {job} failed rc={rc}\nstdout:\n{o[-4000:]}\nstderr:\n{err[-4000:]}"
    return outs
