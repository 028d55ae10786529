"""aligned.log comparisons: the lines that differ from run to run, and the inputs of hostio.summary_log a reference log states."""
import re

_STAMP = re.compile(r"^ \w{3} \w{3} [ \d]\d \d\d:\d\d:\d\d \d{4}$")


def strip_volatile(log: str) -> str:
    """aligned.log without the Command lines (the command and the line under it), the "Process pid" line and the timestamp"""
    out, skip = [], False
    for ln in log.split("\n"):
        if skip:
            skip = False
            continue
        if ln == " Command:":
            skip = True
            continue
        if ln.startswith(" Process pid =") or _STAMP.match(ln):
            continue
        out.append(ln)
    return "\n".join(out)


def log_inputs(log: str) -> dict:
    """what a caller passes summary_log and reads off its own run: lambda / K as printed (6 significant digits) and the minimal
    SW scores per index"""
    return dict(gumbel=[(float(a), float(b)) for a, b in re.findall(r"Gumbel lambda = (\S+)\n\s+Gumbel K = (\S+)", log)],
                minimal_score=[int(x) for x in re.findall(r"Minimal SW score based on E-value = (\d+)", log)])
