"""Launchers: flag → environment mapping, static launcher failure propagation, elastic restart-all semantics
(reference: bagua/distributed/launch.py:157-179,283-300; run.py + torch elastic)."""
import os
import signal
import subprocess
import sys
import textwrap

import pytest

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ENV = dict(os.environ, PYTHONPATH=REPO + os.pathsep + os.environ.get("PYTHONPATH", ""), CUDA_VISIBLE_DEVICES="", BAGUA_FORCE_CPU="1")


def _port():
    from tests.mp_utils import free_port

    return free_port()


def test_set_bagua_env_and_parser():
    from bagua_b200.distributed import launch

    args = launch.parse_args(["--nproc_per_node", "4", "--autotune_level", "1", "--default_bucket_size", "123", "--bagua_service_port", "4242",
                              "--master_addr", "10.0.0.1", "--report_metrics", "train.py", "--lr", "0.1"])
    env = {}
    launch.set_bagua_env(args, env)
    assert env["BAGUA_DEFAULT_BUCKET_SIZE"] == "123" and env["BAGUA_AUTOTUNE"] == "1" and env["BAGUA_SERVICE_PORT"] == "4242"
    assert env["AUTO_TUNE_SERVER_ADDR"] == "10.0.0.1:4242" and env["BAGUA_REPORT_METRICS"] == "1"
    assert args.training_script == "train.py" and args.training_script_args == ["--lr", "0.1"] and "NCCL_NET_PLUGIN" not in env
    args = launch.parse_args(["--enable_bagua_net", "train.py"])
    launch.set_bagua_env(args, env)
    assert env["NCCL_NET_PLUGIN"] == "bagua" and os.path.exists(os.path.join(env["LD_LIBRARY_PATH"].split(":")[0], "libnccl-net-bagua.so"))
    from bagua_b200.distributed import run

    a = run.parse_args(["--standalone", "--nproc_per_node", "2", "--autotune_level", "0", "x.py"])
    assert a.standalone and a.autotune_level == 0


def test_static_launcher_propagates_failure(tmp_path):
    script = tmp_path / "w.py"
    script.write_text(textwrap.dedent("""
        import os, sys, time
        if os.environ["RANK"] == "1":
            sys.exit(3)
        time.sleep(30)
    """))
    from tests.mp_utils import run_in_session

    r = run_in_session([sys.executable, "-m", "bagua_b200.distributed.launch", "--nproc_per_node=2", f"--master_port={_port()}", str(script)], 60, env=ENV)
    assert r.returncode != 0  # the surviving worker was terminated long before its 30 s sleep ended


def test_elastic_launcher_restarts_all_workers(tmp_path):
    marker = tmp_path / "attempts"
    script = tmp_path / "w.py"
    script.write_text(textwrap.dedent(f"""
        import os, sys
        sys.path.insert(0, {REPO!r})
        import torch, bagua_b200 as bagua
        bagua.init_process_group()
        restart = int(os.environ.get("TORCHELASTIC_RESTART_COUNT", "0"))
        with open({str(marker)!r} + f".{{bagua.get_rank()}}.{{restart}}", "w") as f:
            f.write("x")
        t = torch.ones(1)
        bagua.allreduce_inplace(t)
        assert t.item() == bagua.get_world_size()
        if restart == 0 and bagua.get_rank() == 1:
            sys.exit(7)   # first attempt: one worker dies → torch elastic restarts the whole gang
        sys.stdout.write(f"DONE {{bagua.get_rank()}} {{restart}}" + chr(10))   # one write: the two workers share the launcher's stdout
        sys.stdout.flush()
        with open({str(marker)!r} + f".done.{{bagua.get_rank()}}", "w") as f:
            f.write(str(restart))
    """))
    # Every attempt of the gang shares the agent-hosted TCPStore; init_process_group isolates the keys of each attempt (without that a
    # restarted rank read its peer's address of the previous attempt and gloo's connectFullMesh was refused about every second
    # time — the round-1 version of this test had to retry and skip). One run, and it has to pass.
    from tests.mp_utils import run_in_session

    r = run_in_session([sys.executable, "-m", "bagua_b200.distributed.run", "--nnodes=1", "--nproc_per_node=2", "--max_restarts=2",
                        "--rdzv_backend=c10d", f"--rdzv_endpoint=127.0.0.1:{_port()}", "--rdzv_id=elastic_test", "--monitor_interval=1",
                        str(script)], 120, env=ENV)
    assert r.returncode == 0, r.stdout[-1500:] + r.stderr[-3000:]
    files = sorted(os.listdir(tmp_path))
    # both ranks ran the failed first attempt and one restarted attempt (restart-all semantics)
    for rank in (0, 1):
        attempts = sorted(int(f.split(".")[2]) for f in files if f.startswith(f"attempts.{rank}."))
        assert attempts[0] == 0 and len(attempts) >= 2 and attempts[-1] > 0, files
    # completion is judged by the marker files (stdout lines of the two workers may interleave)
    assert all((tmp_path / f"attempts.done.{rank}").exists() for rank in (0, 1)), (files, r.stdout)


def test_workers_die_when_the_launcher_is_killed(tmp_path):
    """SIGKILL the static launcher: its workers must not survive it (PR_SET_PDEATHSIG)."""
    import signal
    import time

    script = tmp_path / "sleepy.py"
    script.write_text("import os, time\nopen(os.environ['PIDFILE'] + os.environ['RANK'], 'w').write(str(os.getpid()))\ntime.sleep(120)\n")
    env = dict(ENV, PIDFILE=str(tmp_path / "pid"))
    proc = subprocess.Popen([sys.executable, "-m", "bagua_b200.distributed.launch", "--nproc_per_node=2", f"--master_port={_port()}", str(script)], env=env,
                            start_new_session=True)
    try:
        deadline = time.time() + 60
        while time.time() < deadline and not all(os.path.exists(str(tmp_path / f"pid{r}")) for r in (0, 1)):
            time.sleep(0.1)
        pids = [int(open(str(tmp_path / f"pid{r}")).read()) for r in (0, 1)]
        os.kill(proc.pid, signal.SIGKILL)
        proc.wait()
        deadline = time.time() + 20
        alive = pids
        while time.time() < deadline and alive:
            alive = [p for p in alive if os.path.exists(f"/proc/{p}") and "zombie" not in open(f"/proc/{p}/status").read().lower()]
            time.sleep(0.2)
        assert not alive, f"workers {alive} outlived the launcher"
    finally:
        try:
            os.killpg(proc.pid, signal.SIGKILL)
        except ProcessLookupError:
            pass


def _fake_ssh(tmp_path):
    """An ``ssh`` that ignores the host and runs the remote command line locally: enough to drive baguarun end to end."""
    d = tmp_path / "bin"
    d.mkdir()
    ssh = d / "ssh"
    ssh.write_text('#!/bin/bash\n# usage: ssh [-o opt] [-p port] host command\nexec bash -c "${@: -1}"\n')
    ssh.chmod(0o755)
    return str(d)


def test_baguarun_starts_one_launcher_per_host_and_propagates_failure(tmp_path):
    from tests.mp_utils import run_in_session

    env = dict(ENV, PATH=_fake_ssh(tmp_path) + os.pathsep + os.environ["PATH"], BAGUA_TEST_MARK="forwarded")
    ok = tmp_path / "ok.py"
    ok.write_text(textwrap.dedent(f"""
        import os, sys
        sys.path.insert(0, {REPO!r})
        import torch, bagua_b200 as bagua
        bagua.init_process_group()
        t = torch.ones(1) * (bagua.get_rank() + 1)
        bagua.allreduce_inplace(t)
        assert t.item() == 3 and bagua.get_world_size() == 2 and os.environ["BAGUA_TEST_MARK"] == "forwarded"
        print("NODE", bagua.get_node_rank(), "OK", flush=True)
    """))
    port = _port()
    r = run_in_session([sys.executable, "-m", "bagua_b200.script.baguarun", "--host_list", "127.0.0.1,localhost", "--nproc_per_node", "1", "--master_port", str(port),
                        "-x", "BAGUA_TEST_MARK", "-x", "PYTHONPATH", "-x", "BAGUA_FORCE_CPU", "-x", "CUDA_VISIBLE_DEVICES", str(ok)], 120, env=env, cwd=str(tmp_path))
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    assert "[127.0.0.1] NODE 0 OK" in r.stdout and "[localhost] NODE 1 OK" in r.stdout
    bad = tmp_path / "bad.py"
    bad.write_text("import os, sys, time\nif os.environ['NODE_RANK'] == '1':\n    sys.exit(5)\ntime.sleep(60)\n")
    r = run_in_session([sys.executable, "-m", "bagua_b200.script.baguarun", "--host_list", "127.0.0.1,localhost", "--nproc_per_node", "1", "--master_port", str(_port()),
                        "-x", "PYTHONPATH", str(bad)], 40, env=env, cwd=str(tmp_path))
    assert r.returncode != 0      # host 1 failed → host 0's 60 s sleep was cut short
    d = subprocess.run([sys.executable, "-m", "bagua_b200.script.baguarun", "--host_list", "a,b,c", "--nproc_per_node", "8", "--dry_run", "train.py", "--lr", "1"],
                       env=env, capture_output=True, text=True)
    lines = d.stdout.strip().splitlines()
    assert len(lines) == 3 and "--nnodes=3" in lines[2] and "--node_rank=2" in lines[2] and "--master_addr=a" in lines[2] and lines[2].rstrip("'").endswith("train.py --lr 1")
    # both --host_list forms, NAME=VALUE exports and the flags that are handed on to the per-host launcher (reference baguarun.py:61-71,176-203)
    d = subprocess.run([sys.executable, "-m", "bagua_b200.script.baguarun", "--host_list", "a:2201,b", "--ssh_port", "2022", "--nproc_per_node", "4", "--dry_run",
                        "--bagua_service_port", "29600", "--no_python", "--enable_bagua_net", "-x", "FOO=bar baz", "-x", "BAGUA_TEST_MARK", "./train.sh", "--lr", "1"],
                       env=env, capture_output=True, text=True)
    lines = d.stdout.strip().splitlines()
    assert len(lines) == 2 and " -p 2201 a " in lines[0] and " -p 2022 b " in lines[1], d.stdout + d.stderr
    for flag in ("--bagua_service_port=29600", "--no_python", "--enable_bagua_net", "--master_addr=a", "FOO=", "bar baz", "BAGUA_TEST_MARK=forwarded"):
        assert flag in lines[1], (flag, lines[1])


def test_bagua_doctor_reports_and_self_tests():
    """``python -m bagua_b200.script.bagua_doctor --json``: library state, versions, environment deviations and a passing self-test."""
    import json
    import subprocess
    import sys

    env = dict(os.environ, NCCL_SOCKET_IFNAME="lo", BAGUA_DEFAULT_BUCKET_SIZE="1048576", CUDA_VISIBLE_DEVICES="")
    r = subprocess.run([sys.executable, "-m", "bagua_b200.script.bagua_doctor", "--json"], capture_output=True, text=True, timeout=180, env=env,
                       cwd=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    rep = json.loads(r.stdout[r.stdout.index("{"):])
    assert rep["ok"] and all(t["ok"] for t in rep["self_test"]) and len(rep["self_test"]) >= 2
    assert rep["libraries"]["_C.so (native core, sm_90a kernels)"]["current_with_sources"] is True
    assert rep["environment"]["BAGUA_DEFAULT_BUCKET_SIZE"] == "1048576" and rep["gpus"]["count"] == 0


def test_bagua_doctor_under_the_launcher_checks_the_collective_path(tmp_path):
    from tests.mp_utils import free_port, run_in_session

    repo = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, NCCL_SOCKET_IFNAME="lo", CUDA_VISIBLE_DEVICES="", BAGUA_FORCE_CPU="1", PYTHONPATH=repo + os.pathsep + os.environ.get("PYTHONPATH", ""))
    r = run_in_session([sys.executable, "-m", "bagua_b200.distributed.launch", "--nproc_per_node=2", f"--master_port={free_port()}", "-m",
                        "bagua_b200.script.bagua_doctor"], 180, env=env, cwd=str(tmp_path))
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert r.stdout.count("[ok] all-reduce across the job: 2 ranks, backend gloo") == 2 and "FAIL" not in r.stdout


def test_elastic_launcher_with_autotune_and_an_unguarded_script(tmp_path):
    """``bagua_b200.distributed.run --standalone --autotune_level 1`` around a training script WITHOUT an ``if __name__ == "__main__"``
    guard (the reference's CI line, .buildkite/scripts/benchmark.sh:14-37): the autotune service must run in its own interpreter
    (a spawn-started multiprocessing child would re-import the script and hang in a second init_process_group) and be reachable
    although the elastic launcher exports the node's hostname — not a routable address in a container — as MASTER_ADDR."""
    from tests.mp_utils import run_in_session

    script = tmp_path / "train.py"
    script.write_text(textwrap.dedent(f"""
        import sys
        sys.path.insert(0, {REPO!r})
        import torch, bagua_b200 as bagua
        from bagua_b200.parallel.algorithms import gradient_allreduce
        bagua.init_process_group()
        assert bagua.communication.get_autotune_service_port() is not None
        torch.manual_seed(0)
        model = torch.nn.Sequential(torch.nn.Linear(64, 256), torch.nn.ReLU(), torch.nn.Linear(256, 256), torch.nn.ReLU(), torch.nn.Linear(256, 8))
        opt = torch.optim.SGD(model.parameters(), lr=0.01)
        model = model.with_bagua([opt], gradient_allreduce.GradientAllReduceAlgorithm())
        sizes = set()
        for it in range(320):
            opt.zero_grad(); model(torch.randn(4, 64)).pow(2).mean().backward(); opt.step()
            sizes.add(model.bagua_ddp._bagua_hyperparameters.bucket_size)
        sys.stdout.write(f"DONE {{bagua.get_rank()}} bucket sizes tried: {{len(sizes)}}" + chr(10)); sys.stdout.flush()
    """))
    env = dict(ENV)
    for k in ("MASTER_ADDR", "MASTER_PORT", "RANK", "WORLD_SIZE"):
        env.pop(k, None)
    r = run_in_session([sys.executable, "-m", "bagua_b200.distributed.run", "--standalone", "--nnodes=1", "--nproc_per_node=2", f"--rdzv_endpoint=127.0.0.1:{_port()}",
                        "--autotune_level", "1", "--autotune_warmup_time", "0", "--autotune_sampling_confidence_time", "0", "--autotune_max_samples", "2",
                        f"--bagua_service_port={_port()}", str(script)], 240, env=env)
    assert r.returncode == 0, r.stdout[-1500:] + r.stderr[-3000:]
    done = [ln for ln in r.stdout.splitlines() if ln.startswith("DONE")]
    assert len(done) == 2 and all(int(ln.rsplit(" ", 1)[1]) >= 2 for ln in done), done   # the service handed out new bucketings
