"""Pins pepper_b200/cli.py's parsers against the UNMODIFIED reference argparse builders and presets: `add_call_variant_arguments`
(pepper_variant/modules/argparse/CallVariantsArguments.py), `set_parameters` (SetParameters.py) and `add_polish_arguments`
(pepper/pepper.py, imported with stand-ins for the pipeline modules it imports but the parser does not use).  Writes
tests/golden/cli_contract.json: for call_variant and polish every option's strings, dest, default, type, action and
`required`; for call_variant and each preset the resolved values of every option on an all-default command line.
    python tests/golden/make_golden_cli.py"""
import argparse
import contextlib
import importlib.util
import io
import json
import os
import sys
import types

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get("PEPPER_REFERENCE", "/root/reference")


def _load(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def _options(p: argparse.ArgumentParser) -> list:
    out = []
    for a in p._actions:
        if isinstance(a, argparse._HelpAction):
            continue
        out.append(dict(option_strings=list(a.option_strings), dest=a.dest, default=a.default,
                        type=a.type.__name__ if a.type is not None else None, action=type(a).__name__, required=bool(a.required)))
    return out


cv = _load("CallVariantsArguments", os.path.join(REF, "pepper_variant/modules/argparse/CallVariantsArguments.py"))
sp = _load("SetParameters", os.path.join(REF, "pepper_variant/modules/argparse/SetParameters.py"))
# pepper.py imports the pipeline modules at the top; add_polish_arguments uses none of them
for name in ("pepper", "pepper.modules", "pepper.modules.python"):
    sys.modules[name] = types.ModuleType(name)
sys.modules["pepper.version"] = types.SimpleNamespace(__version__="0")
for mod, fn in (("polish", "polish"), ("make_images", "make_images"), ("call_consensus", "call_consensus"),
                ("perform_stitch", "perform_stitch"), ("download_model", "download_models")):
    sys.modules["pepper.modules.python." + mod] = types.SimpleNamespace(**{fn: None})
pp = _load("pepper_main", os.path.join(REF, "pepper/pepper.py"))

cv_parser = cv.add_call_variant_arguments(argparse.ArgumentParser())
po_parser = pp.add_polish_arguments(argparse.ArgumentParser())
REQUIRED = ["-b", "r.bam", "-f", "r.fa", "-m", "m.pkl", "-o", "out", "-s", "S", "-t", "4"]
presets = {}
for preset in ("ont_r9_guppy5_sup", "ont_r9_guppy4_hac", "ont_r10_q20", "hifi", "clr"):
    ns = cv_parser.parse_args(REQUIRED + ["--" + preset])
    ns.sub_command = "call_variant"
    with contextlib.redirect_stderr(io.StringIO()):
        ns = sp.set_parameters(ns)
    presets[preset] = {k: v for k, v in sorted(vars(ns).items()) if k != "sub_command"}
out = dict(call_variant=dict(options=_options(cv_parser), required_argv=REQUIRED, presets=presets),
           polish=dict(options=_options(po_parser)))
with open(os.path.join(HERE, "cli_contract.json"), "w") as f:
    json.dump(out, f, indent=1, sort_keys=True)
    f.write("\n")
print("wrote cli_contract.json: %d call_variant options, %d polish options" % (len(out["call_variant"]["options"]),
                                                                           len(out["polish"]["options"])))
