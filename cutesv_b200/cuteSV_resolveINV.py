"""Drop-in for the reference's cuteSV_resolveINV (resolveINV.py:6-99,205-252)."""
from . import _abi, workdir
from ._resolve_common import resolve_one
from .cuteSV_genotype import call_gt_genos, geno_fields


def resolution_INV(path, chr, svtype, read_count, max_cluster_bias, sv_size, bam_path, action, MaxSize, gt_round, sigs_index):
    p = _abi.default_params(min_support=read_count, bias_inv=max_cluster_bias, min_size=sv_size, max_size=MaxSize,
                            genotype=1 if action else 0, gt_round=gt_round)
    return resolve_one(path, chr, "INV", p, sigs_index, action)


def run_inv(args):
    return resolution_INV(*args)


def call_gt(temporary_dir, chr, candidate_single_SV, max_cluster_bias, sigs_index):
    """Genotyped rows of resolveINV.py:208-252: candidates [chr, svtype, bp1, inv_len, support, strand, read names, bp2]; the
    cover sets of the windows bp1 +- max_cluster_bias/2 and bp2 +- max_cluster_bias/2 are united."""
    if chr not in sigs_index["reads"].keys():
        return []
    reads_list = workdir.load_slice(temporary_dir, "reads", chr, sigs_index)
    svs_list = [(max(item[k] - max_cluster_bias / 2, 0), item[k] + max_cluster_bias / 2) for k in (2, 7) for item in candidate_single_SV]
    genos = call_gt_genos(reads_list, svs_list, 2, [item[6] for item in candidate_single_SV])
    out = []
    for item, g in zip(candidate_single_SV, genos):
        dr, gt, gl, gq, qual = geno_fields(g)
        out.append([item[0], item[1], str(int(item[2])), str(int(item[3])), str(item[4]), dr, gt, item[5], gl, gq, qual, ",".join(item[6])])
    return out
