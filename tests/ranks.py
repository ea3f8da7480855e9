"""Launching ranks under torchrun from a test, with nothing left running if they outlive their timeout.

torchrun starts every rank in a session of its own, so killing the launcher's process group does not reach them.  Each
rank therefore records its pid as `pid.<RANK>` in a directory the test names (RANK_PID_LINES does it), and on timeout
the launcher is asked to stop its ranks (SIGTERM, which torchrun passes on), and whatever is still alive after a bounded
wait, launcher or rank, is killed."""
import os
import signal
import subprocess
import sys
import time

# the first lines of a rank's script: its pid, as pid.<RANK> in $SVCB_PID_DIR
RANK_PID_LINES = ("import os\n"
                  "with open(os.path.join(os.environ['SVCB_PID_DIR'], 'pid.' + os.environ['RANK']), 'w') as _f:\n"
                  "    _f.write(str(os.getpid()))\n")
GRACE = 30   # seconds torchrun gets to stop its ranks after SIGTERM


def alive(pid):
    """True while `pid` exists and is not a zombie."""
    try:
        with open(f"/proc/{pid}/stat") as f:
            return f.read().rsplit(")", 1)[1].split()[0] != "Z"
    except (FileNotFoundError, ProcessLookupError, IndexError):
        return False


def ours(pid, pid_dir):
    """True if `pid` is still a rank started with this pid directory (and not a reused pid)."""
    try:
        with open(f"/proc/{pid}/environ", "rb") as f:
            return f"SVCB_PID_DIR={pid_dir}".encode() in f.read().split(b"\0")
    except OSError:
        return False


def rank_pids(pid_dir):
    pids = []
    for name in sorted(os.listdir(pid_dir)):
        if name.startswith("pid."):
            with open(os.path.join(pid_dir, name)) as f:
                text = f.read().strip()
            if text:
                pids.append(int(text))
    return pids


def torchrun(args, nproc, cwd, env, timeout, pid_dir):
    """`python -m torch.distributed.run --standalone --nproc-per-node nproc *args` in cwd; the scripts it runs must
    begin with RANK_PID_LINES.  -> (return code or None on timeout, stdout, stderr).  On timeout the launcher gets
    SIGTERM and GRACE seconds, then it and every recorded rank still alive get SIGKILL."""
    env = dict(env, SVCB_PID_DIR=str(pid_dir))
    p = subprocess.Popen([sys.executable, "-m", "torch.distributed.run", "--standalone", "--nproc-per-node", str(nproc),
                          *args], cwd=cwd, env=env, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True,
                         start_new_session=True)
    try:
        out, err = p.communicate(timeout=timeout)
        return p.returncode, out, err
    except subprocess.TimeoutExpired:
        pass
    p.terminate()
    try:
        out, err = p.communicate(timeout=GRACE)
    except subprocess.TimeoutExpired:
        os.killpg(p.pid, signal.SIGKILL)
        out, err = p.communicate()
    for pid in rank_pids(pid_dir):
        if alive(pid) and ours(pid, pid_dir):
            try:
                os.kill(pid, signal.SIGKILL)
            except ProcessLookupError:
                pass
    deadline = time.monotonic() + GRACE
    while any(alive(pid) for pid in rank_pids(pid_dir)) and time.monotonic() < deadline:
        time.sleep(0.2)
    return None, out, err
