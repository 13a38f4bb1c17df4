"""ORACLE -- test infrastructure only (never imported by detectorch_b200/)."""
import os


def usable_cpus():
    """Host threads this process may really use: the scheduler affinity mask, capped by the cgroup CPU quota (cpu.max) when there is one.
    os.cpu_count() alone counts every core of the machine, and a torch thread pool of that size inside a smaller cgroup quota
    oversubscribes the cores it may use."""
    try:
        n = len(os.sched_getaffinity(0))
    except Exception:
        n = os.cpu_count() or 1
    for path in ("/sys/fs/cgroup/cpu.max", "/sys/fs/cgroup/cpu/cpu.cfs_quota_us"):
        try:
            txt = open(path).read().split()
            if path.endswith("cpu.max"):
                if txt[0] != "max":
                    n = min(n, max(1, int(float(txt[0]) / float(txt[1]))))
            else:
                q = int(txt[0])
                if q > 0:
                    per = int(open("/sys/fs/cgroup/cpu/cpu.cfs_period_us").read())
                    n = min(n, max(1, q // per))
        except Exception:
            pass
    return max(1, n)
