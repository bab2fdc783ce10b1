"""Minimal docopt (reference train.py:24): supports the ``usage: prog [options] <a> <b>`` pattern, whose last
positional may repeat (``<c>...``: one or more, returned as a list), with an ``options:`` section of
``--name=<v>  text [default: x]`` / ``--flag`` / ``-h, --help`` lines."""
import re
import sys


def docopt(doc, argv=None):
    argv = list(sys.argv[1:] if argv is None else argv)
    usage = re.search(r"usage:\s*\S+(.*)", doc, re.I).group(1)
    positional = re.findall(r"<([^>]+)>", usage)
    repeats = bool(re.search(r">\.\.\.", usage))
    opts, takes_value = {}, {}
    in_opts = False
    for line in doc.splitlines():
        if re.match(r"\s*options:", line, re.I):
            in_opts = True
            continue
        if not in_opts:
            continue
        m = re.match(r"\s+(-\w,\s*)?(--[\w-]+)(=<[^>]+>)?", line)
        if not m:
            continue
        name = m.group(2)
        takes_value[name] = m.group(3) is not None
        d = re.search(r"\[default:\s*(.*?)\]", line)
        opts[name] = (d.group(1) if d else None) if takes_value[name] else False
        if m.group(1):
            takes_value[m.group(1).strip(", ")] = False
    args, pos = dict(opts), []
    i = 0
    while i < len(argv):
        a = argv[i]
        if a in ("-h", "--help"):
            print(doc)
            sys.exit(0)
        if a.startswith("--"):
            name, eq, val = a.partition("=")
            if name not in takes_value:
                raise SystemExit("unknown option %s\n%s" % (name, doc))
            if takes_value[name]:
                if not eq:
                    i += 1
                    val = argv[i]
                args[name] = val
            else:
                args[name] = True
        else:
            pos.append(a)
        i += 1
    if len(pos) != len(positional) and not (repeats and len(pos) > len(positional)):
        raise SystemExit(doc)
    for n, v in zip(positional, pos):
        args["<%s>" % n] = v
    if repeats:
        args["<%s>" % positional[-1]] = pos[len(positional) - 1:]
    return args
