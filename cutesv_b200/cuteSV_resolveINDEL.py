"""Drop-in for the reference's cuteSV_resolveINDEL (resolveINDEL.py:17-108, 222-317, 435-479):
same names, same argument meaning, same returned rows -- computed by the CUDA path."""
from . import _abi, workdir
from ._resolve_common import resolve_one
from .cuteSV_genotype import call_gt_genos, geno_fields


def resolution_DEL(path, chr, svtype, read_count, threshold_gloab, max_cluster_bias, minimum_support_reads, bam_path, action,
                   gt_round, remain_reads_ratio, sigs_index):
    p = _abi.default_params(min_support=read_count, min_support_allele=minimum_support_reads, ratio_del=threshold_gloab,
                            bias_del=max_cluster_bias, genotype=1 if action else 0, gt_round=gt_round,
                            remain_reads_ratio=remain_reads_ratio)
    return resolve_one(path, chr, "DEL", p, sigs_index, action)


def resolution_INS(path, chr, svtype, read_count, threshold_gloab, max_cluster_bias, minimum_support_reads, bam_path, action,
                   gt_round, remain_reads_ratio, sigs_index):
    p = _abi.default_params(min_support=read_count, min_support_allele=minimum_support_reads, ratio_ins=threshold_gloab,
                            bias_ins=max_cluster_bias, genotype=1 if action else 0, gt_round=gt_round,
                            remain_reads_ratio=remain_reads_ratio)
    return resolve_one(path, chr, "INS", p, sigs_index, action)


def run_del(args):
    return resolution_DEL(*args)


def run_ins(args):
    return resolution_INS(*args)


def call_gt(temporary_dir, chr, candidate_single_SV, max_cluster_bias, svtype, sigs_index):
    """Genotyped rows of resolveINDEL.py:441-479: candidates [chr, svtype, pos, len, support, CIPOS, CILEN, search position,
    read names(, INS sequence)], DR counted over the window search position +- max_cluster_bias."""
    if chr not in sigs_index["reads"].keys():
        return []
    reads_list = workdir.load_slice(temporary_dir, "reads", chr, sigs_index)
    svs_list = [(max(item[7] - max_cluster_bias, 0), item[7] + max_cluster_bias) for item in candidate_single_SV]
    genos = call_gt_genos(reads_list, svs_list, 1, [item[8] for item in candidate_single_SV])
    out = []
    for item, g in zip(candidate_single_SV, genos):
        row = [item[0], item[1], str(item[2]), str(item[3]), str(item[4]), item[5], item[6]] + list(geno_fields(g)) + [",".join(item[8])]
        if svtype == "INS":
            row.append(item[9])
        out.append(row)
    return out
