"""Drop-in for the reference's cuteSV_resolveDUP (resolveDUP.py:17-77,134-181)."""
from . import _abi, workdir
from ._resolve_common import resolve_one
from .cuteSV_genotype import call_gt_genos, geno_fields


def resolution_DUP(path, chr, read_count, max_cluster_bias, sv_size, bam_path, action, MaxSize, gt_round, sigs_index):
    p = _abi.default_params(min_support=read_count, bias_dup=max_cluster_bias, min_size=sv_size, max_size=MaxSize,
                            genotype=1 if action else 0, gt_round=gt_round)
    return resolve_one(path, chr, "DUP", p, sigs_index, action)


def run_dup(args):
    return resolution_DUP(*args)


def call_gt(temporary_dir, chr, candidate_single_SV, max_cluster_bias, sigs_index):
    """Genotyped rows of resolveDUP.py:137-181: candidates [chr, 'DUP', bp1, bp2, read names]; the cover sets of the windows
    around both breakpoints (half-width min(max_cluster_bias, bp2 - bp1) / 2) are united."""
    if chr not in sigs_index["reads"].keys():
        return []
    reads_list = workdir.load_slice(temporary_dir, "reads", chr, sigs_index)
    svs_list = []
    for k in (2, 3):
        for item in candidate_single_SV:
            nb = min(max_cluster_bias, item[3] - item[2])
            svs_list.append((max(item[k] - nb / 2, 0), item[k] + nb / 2))
    genos = call_gt_genos(reads_list, svs_list, 2, [item[4] for item in candidate_single_SV])
    return [[item[0], item[1], str(item[2]), str(item[3] - item[2]), str(len(item[4]))] + list(geno_fields(g)) + [",".join(item[4])]
            for item, g in zip(candidate_single_SV, genos)]
