"""The platform presets of `call_variant` as data: one table per preset of the values each one gives the image-generation and
candidate-finding options (`pepper_variant` SetParameters.py), and the mapping of a resolved option set onto the arguments of
the device pipelines (image thresholds, candidate options, VCF options, get_reads filters).

A preset only fills an option the user left unset (None); `--skip_indels` given on the command line stays on under every
preset, and `--clr` turns it on."""
from __future__ import annotations

PRESETS = ("ont_r9_guppy5_sup", "ont_r9_guppy4_hac", "ont_r10_q20", "hifi", "clr")

# image generation (make_images): get_reads filters and the encoder's candidate thresholds
IMAGE_KEYS = ("min_mapq", "min_snp_baseq", "min_indel_baseq", "snp_frequency", "insert_frequency", "delete_frequency",
              "min_coverage_threshold", "candidate_support_threshold", "snp_candidate_frequency_threshold",
              "indel_candidate_frequency_threshold", "skip_indels")
# candidate finding (find_candidates): the selection of candidate options and the VCF writer's options
CANDIDATE_KEYS = ("allowed_multiallelics", "snp_p_value", "insert_p_value", "delete_p_value", "snp_q_cutoff", "indel_q_cutoff",
                  "report_snp_above_freq", "report_indel_above_freq", "snp_p_value_in_lc", "insert_p_value_in_lc",
                  "delete_p_value_in_lc", "snp_q_cutoff_in_lc", "indel_q_cutoff_in_lc")


def _table(image: tuple, candidate: tuple) -> dict:
    return dict(zip(IMAGE_KEYS, image)) | dict(zip(CANDIDATE_KEYS, candidate))


# values in the order of IMAGE_KEYS, then of CANDIDATE_KEYS
TABLES = {
    "ont_r9_guppy5_sup": _table((5, 1, 1, 0.10, 0.15, 0.15, 3, 2, 0.10, 0.10, False),
                                (4, 0.1, 0.1, 0.1, 20, 15, 0, 0, 0.1, 0.15, 0.1, 20, 10)),
    "ont_r9_guppy4_hac": _table((5, 1, 1, 0.10, 0.12, 0.12, 3, 2, 0.10, 0.10, False),
                                (4, 0.10, 0.25, 0.25, 20, 15, 0, 0, 0.05, 0.01, 0.01, 20, 10)),
    "ont_r10_q20": _table((1, 1, 1, 0.1, 0.1, 0.1, 3, 2, 0.10, 0.10, False),
                          (4, 0.00001, 0.001, 0.001, 15, 30, 0, 0, 0.000001, 0.001, 0.001, 20, 35)),
    "hifi": _table((5, 10, 10, 0.10, 0.12, 0.10, 2, 2, 0.10, 0.10, False),
                   (4, 0, 0, 0, 15, 20, 0, 0, 0, 0, 0, 15, 20)),
    "clr": _table((5, 0, 0, 0.10, 0.12, 0.12, 3, 2, 0.10, 0.12, True),
                  (4, 0.1, 0.2, 0.2, 20, 20, 0, 0, 0.05, 0.05, 0.05, 20, 20)),
}


def resolve(preset: str, given: dict) -> dict:
    """The option values of `preset` with every option of `given` that is not None kept (skip_indels: kept when True)."""
    out = dict(given)
    for k, v in TABLES[preset].items():
        if k == "skip_indels":
            out[k] = bool(given.get(k)) or v
        elif given.get(k) is None:
            out[k] = v
    return out


def image_params(o: dict) -> dict:
    """Resolved options -> the `params` of the variant encoder (the keys of synth.ont_params())."""
    return dict(min_snp_baseq=int(o["min_snp_baseq"]), min_indel_baseq=int(o["min_indel_baseq"]),
                snp_freq_threshold=float(o["snp_frequency"]), insert_freq_threshold=float(o["insert_frequency"]),
                delete_freq_threshold=float(o["delete_frequency"]), min_coverage_threshold=int(o["min_coverage_threshold"]),
                snp_candidate_freq_threshold=float(o["snp_candidate_frequency_threshold"]),
                indel_candidate_freq_threshold=float(o["indel_candidate_frequency_threshold"]),
                candidate_support_threshold=int(o["candidate_support_threshold"]), skip_indels=int(bool(o["skip_indels"])))


def candidate_options(o: dict) -> dict:
    """Resolved options -> the candidate selection's options (candidates.PbCandidateOptions fields, as candidates.ONT_OPTIONS)."""
    from .candidates import PbCandidateOptions
    return {k: float(o[k]) for k, _ in PbCandidateOptions._fields_}


def vcf_options(o: dict) -> dict:
    """Resolved options -> the VCF writer's options (as vcf.VCF_OPTIONS_ONT)."""
    return dict(allowed_multiallelics=int(o["allowed_multiallelics"]),
                **{k: float(o[k]) for k in ("snp_q_cutoff", "indel_q_cutoff", "snp_q_cutoff_in_lc", "indel_q_cutoff_in_lc")})


def read_filters(o: dict) -> dict:
    """Resolved options -> the get_reads filters of the variant read source."""
    return dict(min_mapq=int(o["min_mapq"]), include_supplementary=bool(o["include_supplementary"]),
                downsample_rate=float(o["downsample_rate"]))
