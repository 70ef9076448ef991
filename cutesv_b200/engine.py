"""Engine: one csv_ctx (one GPU) driven from Python.  Host side of the drop-in boundary."""
import ctypes as C

import numpy as np

from . import _abi, _lib


class Engine(object):
    """Owns a csv_ctx.  stream: optional cudaStream_t handle (e.g. torch.cuda.current_stream().cuda_stream)."""

    def __init__(self, device=0, stream=None, params=None, contig_lens=None):
        self.L = _lib.lib()
        h = C.c_void_p()
        _lib.check(self.L.csv_create(int(device), C.c_void_p(stream) if stream else None, C.byref(h)))
        self.h = h
        self.device = int(device)
        self.params = None
        self._keep = None
        self.set_params(params if params is not None else _abi.default_params())
        if contig_lens is not None:
            self.set_contigs(contig_lens)

    def close(self):
        if getattr(self, "h", None):
            self.L.csv_destroy(self.h)
            self.h = None
        for p in getattr(self, "_pinned", []):
            self.L.csv_host_free(p)
        self._pinned = []

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_params(self, params):
        self.params = params
        _lib.check(self.L.csv_set_params(self.h, C.byref(params)))

    def set_contigs(self, lens, names=None):
        """Contig table (csv_set_contigs); names (str or bytes per contig id, optional): the contig names that SA:Z text reduced on
        the device (reduce_sa, packets with sa_text) is matched against (csv_set_contig_names)."""
        lens = np.ascontiguousarray(lens, dtype=np.int64)
        self.n_contigs = len(lens)
        _lib.check(self.L.csv_set_contigs(self.h, C.c_int32(len(lens)), lens.ctypes.data_as(C.POINTER(C.c_int64))))
        if names is not None:
            enc = [nm.encode() if isinstance(nm, str) else bytes(nm) for nm in names]
            off = np.zeros(len(enc) + 1, dtype=np.int64)
            np.cumsum([len(b) for b in enc], out=off[1:])
            raw = np.frombuffer(b"".join(enc) or b"\0", dtype=np.uint8)
            _lib.check(self.L.csv_set_contig_names(self.h, C.c_int32(len(enc)), raw.ctypes.data_as(C.POINTER(C.c_uint8)),
                                                   off.ctypes.data_as(C.POINTER(C.c_int64))))

    def set_profiling(self, on):
        """True: every launch between CUDA events.  "lanes": only the INS / DEL back-end intervals and the
        serial tail after the lane join ("tail"), launches as unprofiled."""
        _lib.check(self.L.csv_set_profiling(self.h, 2 if on == "lanes" else int(bool(on))))

    def set_lanes(self, on):
        """Per-SV-type stream lanes (default on); off serialises the types on the ctx stream."""
        _lib.check(self.L.csv_set_lanes(self.h, int(bool(on))))

    # -- device-resident path (bench `value`): upload once, cluster many times --

    def _producer_stream(self, stream, groups):
        """cudaStream_t of device uploads: `stream` (a handle or a torch.cuda.Stream); else torch's current stream on the engine's
        device when a column is a torch tensor; else 0 (the legacy default stream)."""
        if stream is not None:
            return int(getattr(stream, "cuda_stream", stream))
        for cols in groups:
            for v in (cols or {}).values():
                if _abi.is_device_array(v) and type(v).__module__.startswith("torch"):
                    import torch
                    return int(torch.cuda.current_stream(self.device).cuda_stream)
        return 0

    def _upload_device(self, t, d, stream):
        """csv_upload_*_device of one normalised column set (_abi.device_cols); t = SV type id, or None for the reads table."""
        s, off = d
        st = C.c_void_p(stream or None)
        if t is None:
            if off is not None:
                _lib.check(self.L.csv_upload_reads_grouped_device(self.h, C.byref(s), off, st))
            else:
                _lib.check(self.L.csv_upload_reads_device(self.h, C.byref(s), st))
        elif off is not None:
            _lib.check(self.L.csv_upload_sigs_grouped_device(self.h, t, C.byref(s), off, st))
        else:
            _lib.check(self.L.csv_upload_sigs_device(self.h, t, C.byref(s), st))

    def upload(self, sigs, reads, grouped=False, stream=None):
        """Asynchronous H2D of the inputs of cluster_device().  grouped=True: dicts from _abi.group_by_contig (rows grouped by
        contig + `contig_off` instead of the contig column; csv_upload_*_grouped).
        Column dicts whose arrays expose __cuda_array_interface__ (torch CUDA tensors) are copied device-to-device instead
        (csv_upload_*_device), in the order of `stream` (see _producer_stream): the copies follow the work already enqueued on it,
        and work enqueued on it after this call (overwriting or freeing the tensors) follows the copies.  One dict is all device
        or all host; device signatures with host reads (or the reverse) are fine."""
        n_contigs = getattr(self, "n_contigs", None)
        dev = {name: _abi.device_cols(sigs.get(name), _abi.SIG_FIELDS, self.device, grouped, n_contigs) for name in _abi.TYPE_NAMES}
        dev_r = _abi.device_cols(reads, _abi.READS_FIELDS, self.device, grouped, n_contigs)
        st = self._producer_stream(stream, list(sigs.values()) + [reads]) if dev_r or any(dev.values()) else 0
        keep = []
        for t, name in enumerate(_abi.TYPE_NAMES):
            if dev[name] is not None:
                self._upload_device(t, dev[name], st)
            elif grouped:
                s, off, k = _abi.make_sig_cols_grouped(sigs.get(name))
                keep.append((k, off))
                if off is not None:
                    _lib.check(self.L.csv_upload_sigs_grouped(self.h, t, C.byref(s), off.ctypes.data_as(C.POINTER(C.c_int64))))
                else:
                    _lib.check(self.L.csv_upload_sigs(self.h, t, C.byref(s)))
            else:
                s, k = _abi.make_sig_cols(sigs.get(name))
                keep.append(k)
                _lib.check(self.L.csv_upload_sigs(self.h, t, C.byref(s)))
        if dev_r is not None:
            self._upload_device(None, dev_r, st)
        elif grouped:
            r, r_off, rk = _abi.make_reads_cols_grouped(reads)
            keep.append((rk, r_off))
            if r_off is not None:
                _lib.check(self.L.csv_upload_reads_grouped(self.h, C.byref(r), r_off.ctypes.data_as(C.POINTER(C.c_int64))))
            else:
                _lib.check(self.L.csv_upload_reads(self.h, C.byref(r)))
        else:
            r, rk = _abi.make_reads_cols(reads)
            keep.append(rk)
            _lib.check(self.L.csv_upload_reads(self.h, C.byref(r)))
        self._keep = keep  # host buffers must outlive the async copies
        self._dev_rows = [len((sigs.get(n) or {}).get("a", ())) for n in _abi.TYPE_NAMES] + [0 if reads is None else len(reads["start"])]

    def upload_alignments(self, aln, stream=None):
        """ALL alignment records in BAM order (dict like the reads table, is_primary = flag in (0, 16)): enables the
        device TRA genotyper (call_gt, resolveTRA.py:260-309).  None / empty clears the table.  Device columns (torch CUDA
        tensors) go through csv_upload_alignments_device in the order of `stream`, as in upload()."""
        d = _abi.device_cols(aln, _abi.READS_FIELDS, self.device)
        if d is not None:
            st = self._producer_stream(stream, [aln])
            _lib.check(self.L.csv_upload_alignments_device(self.h, C.byref(d[0]), C.c_void_p(st or None)))
            self._keep_aln = ()
            return
        r, keep = _abi.make_reads_cols(aln)
        _lib.check(self.L.csv_upload_alignments(self.h, C.byref(r)))
        self._keep_aln = keep

    def cluster_device(self, type_mask=0x1F):
        _lib.check(self.L.csv_cluster(self.h, C.c_uint32(type_mask)))

    def result_tensors(self):
        """Zero-copy torch views of the last cluster call's results on the engine's device (csv_result_device_ptrs):
        (cands [n, 16] int32 = csv_cand, genos [n, 10] int32 = csv_geno (qual is the float64 in words 8-9), names int32).
        Blocks until the results are ready.  The views alias the engine's own buffers: they are valid until the next upload,
        cluster call or close() on this engine, so clone() whatever you keep."""
        import torch
        nc, nn = self.counts()
        a, b, c = self.device_ptrs()
        dev = torch.device("cuda", self.device)
        return (torch.as_tensor(_DeviceView(a, (nc, 16)), device=dev), torch.as_tensor(_DeviceView(b, (nc, 10)), device=dev),
                torch.as_tensor(_DeviceView(c, (nn,)), device=dev))

    def counts(self):
        nc, nn = C.c_int64(0), C.c_int64(0)
        _lib.check(self.L.csv_result_counts(self.h, C.byref(nc), C.byref(nn)))
        return nc.value, nn.value

    def fetch(self, out=None):
        nc, nn = self.counts()
        if out is not None:
            cands, genos, names = out
        else:
            cands = np.zeros(max(nc, 1), dtype=_abi.CAND_DTYPE)
            genos = np.zeros(max(nc, 1), dtype=_abi.GENO_DTYPE)
            names = np.zeros(max(nn, 1), dtype=np.int32)
        _lib.check(self.L.csv_fetch(self.h, cands.ctypes.data_as(C.c_void_p), genos.ctypes.data_as(C.c_void_p), C.c_int64(len(cands)),
                                    _abi.ptr(names), C.c_int64(len(names))))
        return cands[:nc], genos[:nc], names[:nn]

    # -- the reference-facing one-shot call: host columns in, host rows out --
    def cluster(self, sigs, reads, type_mask=0x1F, out=None, grouped=False, stream=None):
        """sigs: {type_name: dict(chrom,a,b,read_id[,c])}; reads: dict(chrom,start,end,read_id,is_primary).
        grouped=True: every dict holds rows grouped by contig and `contig_off` instead of `chrom`
        (_abi.group_by_contig; csv_cluster_host_grouped).
        Returns (cands, genos, names) numpy arrays in the reference's emission order.
        When any dict holds device columns (torch CUDA tensors), the inputs go through upload(..., stream=stream) and
        csv_cluster instead of csv_cluster_host; the records still come back to the host."""
        if any(_abi.is_device_array(v) for cols in list(sigs.values()) + [reads] for v in (cols or {}).values()):
            self.upload({k: v for k, v in sigs.items() if type_mask >> _abi.TYPE_IDS[k] & 1}, reads, grouped=grouped, stream=stream)
            self.cluster_device(type_mask)
            return self.fetch(out)
        arr = (_abi.csv_sig_cols * _abi.CSV_NTYPES)()
        offs = (C.POINTER(C.c_int64) * _abi.CSV_NTYPES)()
        keep = []
        total = 0
        for t, name in enumerate(_abi.TYPE_NAMES):
            if grouped:
                s, off, k = _abi.make_sig_cols_grouped(sigs.get(name))
                if off is not None:
                    offs[t] = off.ctypes.data_as(C.POINTER(C.c_int64))
            else:
                s, k = _abi.make_sig_cols(sigs.get(name))
            arr[t] = s
            keep.append(k)
            total += s.n
        if grouped:
            r, r_off, rk = _abi.make_reads_cols_grouped(reads)
        else:
            r, rk = _abi.make_reads_cols(reads)
        if out is None:
            cap_c = max(2 * (total // max(min(self.params.min_support_allele, self.params.min_support), 1)) + 16, 16)
            cap_n = total + 16
            cands = np.zeros(cap_c, dtype=_abi.CAND_DTYPE)
            genos = np.zeros(cap_c, dtype=_abi.GENO_DTYPE)
            names = np.zeros(cap_n, dtype=np.int32)
        else:
            cands, genos, names = out
        nc, nn = C.c_int64(0), C.c_int64(0)
        tail = (C.c_uint32(type_mask), cands.ctypes.data_as(C.c_void_p), genos.ctypes.data_as(C.c_void_p), C.c_int64(len(cands)),
                _abi.ptr(names), C.c_int64(len(names)), C.byref(nc), C.byref(nn))
        self._dev_rows = [int(arr[t].n) for t in range(_abi.CSV_NTYPES)] + [int(r.n)]
        if grouped:
            _lib.check(self.L.csv_cluster_host_grouped(self.h, arr, offs, C.byref(r),
                                                       None if r_off is None else r_off.ctypes.data_as(C.POINTER(C.c_int64)), *tail))
        else:
            _lib.check(self.L.csv_cluster_host(self.h, arr, C.byref(r), *tail))
        return cands[:nc.value], genos[:nc.value], names[:nn.value]

    def cal_gl(self, c0, c1):
        c0 = np.ascontiguousarray(c0, dtype=np.int32)
        c1 = np.ascontiguousarray(c1, dtype=np.int32)
        out = np.zeros(len(c0), dtype=_abi.GENO_DTYPE)
        _lib.check(self.L.csv_cal_gl(self.h, _abi.ptr(c0), _abi.ptr(c1), C.c_int64(len(c0)), out.ctypes.data_as(C.c_void_p)))
        return out

    def overlap_cover(self, windows, reads=None, overlap=True):
        """overlap_cover (cuteSV_genotype.py:95-159) on the device.  windows: _abi.WINDOW_DTYPE array (half units); reads: dict
        (chrom, start, end, read_id, is_primary) or None for the device-resident reads table.  Returns dict(iteration, primary_num,
        cover_off, cover_ids[, overlap_off, overlap_ids]): per window the overlapping rows, the overlapping primary rows and the
        ascending distinct read ids of the primary covering / overlapping rows as CSR."""
        w = np.ascontiguousarray(windows, dtype=_abi.WINDOW_DTYPE)
        n = len(w)
        r, keep = _abi.make_reads_cols(reads) if reads is not None else (None, ())
        it = np.zeros(max(n, 1), np.int32)
        pn = np.zeros(max(n, 1), np.int32)
        co = np.zeros(n + 1, np.int64)
        oo = np.zeros(n + 1, np.int64)
        cap_c = cap_o = 4 * n + 1024
        nc, no = C.c_int64(0), C.c_int64(0)
        while True:
            ci = np.zeros(cap_c, np.int32)
            oi = np.zeros(cap_o, np.int32) if overlap else None
            rc = self.L.csv_overlap_cover(self.h, w.ctypes.data_as(C.c_void_p), C.c_int64(n), C.byref(r) if r is not None else None, _abi.ptr(it),
                                          _abi.ptr(pn), co.ctypes.data_as(C.POINTER(C.c_int64)), _abi.ptr(ci), C.c_int64(cap_c),
                                          oo.ctypes.data_as(C.POINTER(C.c_int64)), _abi.ptr(oi), C.c_int64(cap_o if overlap else 0),
                                          C.byref(nc), C.byref(no))
            if rc != _abi.CSV_E_CAPACITY:
                break
            cap_c, cap_o = max(cap_c, nc.value), max(cap_o, no.value)
        _lib.check(rc)
        del keep
        out = dict(iteration=it[:n], primary_num=pn[:n], cover_off=co, cover_ids=ci[:nc.value])
        if overlap:
            out.update(overlap_off=oo, overlap_ids=oi[:no.value])
        return out

    def call_gt(self, windows, windows_per_cand, support_off, support_ids, reads=None):
        """call_gt + assign_gt (resolveINDEL.py:441, resolveDUP.py:137, resolveINV.py:208) on the device: candidate i owns windows
        [i*windows_per_cand, (i+1)*windows_per_cand) (united cover sets) and support ids [support_off[i], support_off[i+1]).
        Returns a GENO_DTYPE array: cal_GL(DR, DV) with dr / dv."""
        w = np.ascontiguousarray(windows, dtype=_abi.WINDOW_DTYPE)
        so = np.ascontiguousarray(support_off, dtype=np.int64)
        si = np.ascontiguousarray(support_ids, dtype=np.int32)
        n = len(so) - 1
        assert len(w) == n * windows_per_cand
        r, keep = _abi.make_reads_cols(reads) if reads is not None else (None, ())
        out = np.zeros(max(n, 1), dtype=_abi.GENO_DTYPE)
        _lib.check(self.L.csv_call_gt(self.h, w.ctypes.data_as(C.c_void_p), C.c_int64(n), C.c_int32(windows_per_cand),
                                      C.byref(r) if r is not None else None, so.ctypes.data_as(C.POINTER(C.c_int64)), _abi.ptr(si),
                                      out.ctypes.data_as(C.c_void_p)))
        del keep
        return out[:n]

    def tra_call_gt(self, queries, support_off, support_ids, bias, gt_round, aln=None):
        """call_gt of resolveTRA.py:260-309 on the device for caller-given breakpoint pairs (_abi.TRA_QUERY_DTYPE; contig ids of the
        set_contigs table, whose lengths clamp the windows).  Query i's supporting read ids are support_ids[support_off[i]:support_off[i+1]]
        (DV = their count).  aln: host all-alignments columns in BAM order (dict like the reads table), or None for the table
        installed by upload_alignments / rank_names.  Returns a GENO_DTYPE array: cal_GL(DR, DV) with dr / dv, or status 2 with
        dr = gt = -1 where the first window's scan returns -1."""
        q = np.ascontiguousarray(queries, dtype=_abi.TRA_QUERY_DTYPE)
        so = np.ascontiguousarray(support_off, dtype=np.int64)
        si = np.ascontiguousarray(support_ids, dtype=np.int32)
        n = len(q)
        assert len(so) == n + 1
        r, keep = _abi.make_reads_cols(aln) if aln is not None else (None, ())
        out = np.zeros(max(n, 1), dtype=_abi.GENO_DTYPE)
        _lib.check(self.L.csv_tra_call_gt(self.h, q.ctypes.data_as(C.c_void_p), C.c_int64(n), C.byref(r) if r is not None else None,
                                          C.c_int32(bias), C.c_int32(gt_round), so.ctypes.data_as(C.POINTER(C.c_int64)), _abi.ptr(si),
                                          out.ctypes.data_as(C.c_void_p)))
        del keep
        return out[:n]

    def sort_sigs(self, svtype):
        """Sort + adjacent de-duplication of process_process_sigs_type (cuteSV:750-857, 958-969) over the device-resident
        columns of one type (name or id) or of the reads table ("reads").  Returns dict(order, contig_off, ins_tie): the input
        rows kept, in the reference's order; the row range of every contig id inside `order` (n_contigs + 1 offsets); for INS
        the flags of rows that tie with their predecessor up to the sequence (zeros for the other types)."""
        t = _abi.CSV_SORT_READS if svtype == "reads" else (_abi.TYPE_IDS[svtype] if isinstance(svtype, str) else int(svtype))
        off = np.zeros(self.n_contigs + 1, np.int64)
        nk = C.c_int64(0)
        # the device-resident row count bounds the kept rows: one call, no capacity retry
        cap = self._dev_rows[t] if getattr(self, "_dev_rows", None) is not None else 0
        while True:
            order = np.zeros(max(cap, 1), np.int64)
            tie = np.zeros(max(cap, 1), np.uint8)
            rc = self.L.csv_sort_sigs(self.h, C.c_int(t), order.ctypes.data_as(C.POINTER(C.c_int64)), C.c_int64(cap), C.byref(nk),
                                      off.ctypes.data_as(C.POINTER(C.c_int64)), tie.ctypes.data_as(C.POINTER(C.c_uint8)))
            if rc != _abi.CSV_E_CAPACITY:
                break
            cap = nk.value
        _lib.check(rc)
        n = nk.value
        return dict(order=order[:n], contig_off=off, ins_tie=tie[:n])

    def set_extract_records(self, on):
        """Store the record index of every row of the following extract() calls (csv_extract_records), for fetch_records."""
        _lib.check(self.L.csv_extract_records(self.h, int(bool(on))))

    def fetch_records(self, svtype, first=0, count=None):
        """Record index of extracted rows [first, first + count) of one type or of the reads table ("reads") (csv_fetch_records)."""
        t = _abi.CSV_SORT_READS if svtype == "reads" else (_abi.TYPE_IDS[svtype] if isinstance(svtype, str) else int(svtype))
        if count is None:
            count = (self._ex_rows if t == _abi.CSV_SORT_READS else self._ex_counts[t]) - first
        out = np.zeros(max(count, 1), np.int32)
        _lib.check(self.L.csv_fetch_records(self.h, C.c_int(t), C.c_int64(first), C.c_int64(count), _abi.ptr(out)))
        return out[:count]

    def stage_ms(self):
        ms = (C.c_float * _abi.CSV_ST_COUNT)()
        _lib.check(self.L.csv_stage_ms(self.h, ms))
        return {name: float(ms[i]) for i, name in enumerate(_abi.STAGES)}

    def sort_probe(self):
        ms, b, n = C.c_float(0), C.c_int64(0), C.c_int32(0)
        _lib.check(self.L.csv_sort_probe(self.h, C.byref(ms), C.byref(b), C.byref(n)))
        return dict(ms=float(ms.value), bytes=int(b.value), launches=int(n.value))

    def counters(self):
        out = (C.c_uint32 * 32)()
        _lib.check(self.L.csv_debug_counters(self.h, out))
        v = list(out)
        t = _abi.TYPE_NAMES
        return dict(status=v[0], n_cand=v[1], n_names=v[2], max_support=v[3], kept=dict(zip(t, v[4:9])), big=dict(zip(t, v[9:14])),
                    giant=dict(zip(t, v[14:19])), pairs=v[19], domain=dict(zip(t, v[20:25])), members=dict(zip(t, v[25:30])), small_path=v[30])

    def kernel_times(self):
        """{kernel name: (launches, total ms)} of the calls made while profiling was on (collected by fetch())."""
        need = int(self.L.csv_kernel_times(self.h, None, 0))
        buf = C.create_string_buffer(need + 16)
        self.L.csv_kernel_times(self.h, buf, need + 16)
        out = {}
        for ln in buf.value.decode().splitlines():
            nm, n, ms = ln.split("\t")
            out[nm] = (int(n), float(ms))
        return out

    def launch_count(self):
        return int(self.L.csv_launch_count(self.h))

    def graph_replays(self):
        return int(self.L.csv_graph_replays(self.h))

    # -- multi-GPU: contig shards + one NCCL all-gather of the final records --

    def set_shard(self, owned):
        """owned: bool/uint8 mask over contig ids (None = all contigs)."""
        if owned is None:
            _lib.check(self.L.csv_set_shard(self.h, None))
            return
        m = np.ascontiguousarray(owned, dtype=np.uint8)
        assert len(m) == self.n_contigs
        _lib.check(self.L.csv_set_shard(self.h, m.ctypes.data_as(C.POINTER(C.c_uint8))))

    def comm_unique_id(self):
        buf = C.create_string_buffer(128)
        _lib.check(self.L.csv_comm_unique_id(buf, 128))
        return buf.raw

    def comm_init(self, uid, rank, world):
        buf = C.create_string_buffer(bytes(uid), 128)
        _lib.check(self.L.csv_comm_init(self.h, buf, int(rank), int(world)))
        self.rank, self.world = int(rank), int(world)

    def comm_destroy(self):
        _lib.check(self.L.csv_comm_destroy(self.h))

    def allgather(self):
        """Asynchronous, collective: pack + ONE ncclAllGather + device merge of the records of the last cluster_device()."""
        _lib.check(self.L.csv_allgather(self.h))

    def set_gather(self, peer_to_peer):
        """True: store into the peers' mail boxes over NVLink (CUDA IPC); False: ncclAllGather."""
        _lib.check(self.L.csv_set_gather(self.h, 1 if peer_to_peer else 0))

    def gather_mode(self):
        return "peer-to-peer" if self.L.csv_gather_mode(self.h) else "nccl"

    def gathered_counts(self):
        nc, nn = C.c_int64(0), C.c_int64(0)
        _lib.check(self.L.csv_gathered_counts(self.h, C.byref(nc), C.byref(nn)))
        return nc.value, nn.value

    def fetch_gathered(self, out=None):
        nc, nn = self.gathered_counts()
        if out is not None:
            cands, genos, names = out
        else:
            cands = np.zeros(max(nc, 1), dtype=_abi.CAND_DTYPE)
            genos = np.zeros(max(nc, 1), dtype=_abi.GENO_DTYPE)
            names = np.zeros(max(nn, 1), dtype=np.int32)
        _lib.check(self.L.csv_fetch_gathered(self.h, cands.ctypes.data_as(C.c_void_p), genos.ctypes.data_as(C.c_void_p), C.c_int64(len(cands)),
                                             _abi.ptr(names), C.c_int64(len(names))))
        return cands[:nc], genos[:nc], names[:nn]

    def device_ptrs(self):
        a, b, c = C.c_void_p(), C.c_void_p(), C.c_void_p()
        _lib.check(self.L.csv_result_device_ptrs(self.h, C.byref(a), C.byref(b), C.byref(c)))
        return a.value, b.value, c.value

    def pin_packet(self, packed):
        """Copy of an alignment packet in page-locked host memory (csv_host_alloc), so that csv_extract's H2D copies run at PCIe
        speed and asynchronously.  The buffers are freed by close()."""
        if not hasattr(self, "_pinned"):
            self._pinned = []

        def pin(a):
            a = np.ascontiguousarray(a)
            p = C.c_void_p()
            _lib.check(self.L.csv_host_alloc(C.byref(p), C.c_size_t(max(a.nbytes, 1))))
            self._pinned.append(p)
            buf = (C.c_char * max(a.nbytes, 1)).from_address(p.value)
            out = np.frombuffer(buf, dtype=a.dtype, count=a.size).reshape(a.shape)
            out[...] = a
            return out

        out = {}
        for k, v in packed.items():
            if k == "sa":
                out[k] = {kk: pin(np.asarray(vv, dtype=np.int32)) for kk, vv in v.items()}
            elif k in ("cigar_off", "sa_off"):
                out[k] = pin(np.asarray(v, dtype=np.int64))
            elif k == "cigar":
                out[k] = pin(np.asarray(v, dtype=np.uint32))
            elif isinstance(v, np.ndarray) and v.dtype.kind in "iu" and k in ("chrom", "ref_start", "ref_end", "flag", "mapq", "query_len", "read_id"):
                out[k] = pin(np.asarray(v, dtype=np.int32))
            else:
                out[k] = v
        return out

    def extract(self, packed, append=False, stream=None):
        """csv_extract on a packing.pack_alignments() packet.  The extracted signatures and reads rows
        stay device-resident as the inputs of cluster_device(); returns dict(counts, n_rows).
        append=True (csv_extract_append): this packet's output is appended to what earlier packets left on the device;
        counts / n_rows are the totals so far and `first` holds the totals before this packet.
        A packet whose arrays expose __cuda_array_interface__ (torch CUDA tensors; see _abi.device_packet) goes through
        csv_extract*_device in the order of `stream` (see _producer_stream), and with seq_off / seq4 (BAM's packed bases) the INS
        sequences are built on the device (fetch_ins_seqs, ins_seq_tensors).  Device and host packets may be mixed in one
        append accumulation.  A device packet with names / name_off (the records' read names as bytes, instead of read_id) goes
        through csv_extract*_named_device: every packet of the accumulation then carries names, and rank_names() turns the
        provisional ids (record indices) into name ranks.  A device packet with sa_text / sa_text_off (the records' SA:Z values as
        text) has them reduced on the device first (reduce_sa; needs set_contigs(..., names))."""
        counts = (C.c_int64 * _abi.CSV_NTYPES)()
        n_rows = C.c_int64(0)
        d = _abi.device_packet(packed, self.device)
        if d is not None:
            rc_, cig_p, n_cig, sa_, seq = d
            st = self._producer_stream(stream, [packed])
            self._reduce_packet_sa(d, st)
            seq_p = C.byref(seq) if seq is not None else None
            if d.names is not None:
                fn = self.L.csv_extract_append_named_device if append else self.L.csv_extract_named_device
                _lib.check(fn(self.h, C.byref(rc_), cig_p, C.c_int64(n_cig), C.byref(sa_), seq_p, C.byref(d.names), C.c_void_p(st or None), counts,
                              C.byref(n_rows)))
            else:
                fn = self.L.csv_extract_append_device if append else self.L.csv_extract_device
                _lib.check(fn(self.h, C.byref(rc_), cig_p, C.c_int64(n_cig), C.byref(sa_), seq_p, C.c_void_p(st or None), counts, C.byref(n_rows)))
        else:
            n = len(packed["chrom"])
            keep = [np.ascontiguousarray(packed[k], dtype=np.int32) for k in ("chrom", "ref_start", "ref_end", "flag", "mapq", "query_len", "read_id")]
            co = np.ascontiguousarray(packed["cigar_off"], dtype=np.int64)
            so = np.ascontiguousarray(packed["sa_off"], dtype=np.int64)
            rc_ = _abi.csv_read_cols(n, *[_abi.ptr(k) for k in keep], co.ctypes.data_as(C.POINTER(C.c_int64)), so.ctypes.data_as(C.POINTER(C.c_int64)))
            sa = {k: np.ascontiguousarray(v, dtype=np.int32) for k, v in packed["sa"].items()}
            sa_ = _abi.csv_sa_cols(len(sa["chrom"]), *[_abi.ptr(sa[k]) for k in ("chrom", "pos0", "strand", "mapq", "first_clip", "last_clip", "ref_span")])
            cig = np.ascontiguousarray(packed["cigar"], dtype=np.uint32)
            fn = self.L.csv_extract_append if append else self.L.csv_extract
            _lib.check(fn(self.h, C.byref(rc_), cig.ctypes.data_as(C.POINTER(C.c_uint32)), C.c_int64(len(cig)), C.byref(sa_), counts, C.byref(n_rows)))
        return self._extracted(counts, n_rows, append)

    def _extracted(self, counts, n_rows, append):
        """Bookkeeping after an extraction call and extract()'s result.  `first*`: the totals before this packet, which the
        mirrors still hold when the packet joined the open accumulation."""
        joined = append and getattr(self, "_ex_appending", False)
        first = self._ex_counts if joined else [0] * _abi.CSV_NTYPES
        first_rows = self._ex_rows if joined else 0
        first_pieces = self._ex_pieces if joined else 0
        self._ex_counts = [int(x) for x in counts]
        self._ex_rows = int(n_rows.value)
        self._dev_rows = self._ex_counts + [self._ex_rows]
        self._ex_appending = bool(append)
        npz = C.c_int64(0)
        _lib.check(self.L.csv_fetch_pieces(self.h, C.c_int64(0), None, C.byref(npz)))
        self._ex_pieces = int(npz.value)
        return dict(counts={name: int(counts[t]) for t, name in enumerate(_abi.TYPE_NAMES)}, n_rows=int(n_rows.value),
                    first={name: first[t] for t, name in enumerate(_abi.TYPE_NAMES)}, first_rows=first_rows, first_pieces=first_pieces,
                    n_pieces=self._ex_pieces)

    def set_scan_regions(self, tasks, bed, chrom_id):
        """Region table of the following scan() calls (csv_set_scan_regions) from cli.task_windows' tasks, cli.load_bed's region lists
        and the contig ids; bed None clears it.  With a table, scan() extracts only the records the CLI keeps with -include_bed."""
        n, win_off, win_start, reg_off, reg = _abi.scan_regions(tasks, bed, chrom_id)
        if n == 0:
            _lib.check(self.L.csv_set_scan_regions(self.h, C.c_int32(0), None, None, None, None))
            return
        _lib.check(self.L.csv_set_scan_regions(self.h, C.c_int32(n), win_off.ctypes.data_as(C.POINTER(C.c_int64)),
                                               win_start.ctypes.data_as(C.POINTER(C.c_double)), reg_off.ctypes.data_as(C.POINTER(C.c_int64)),
                                               reg.ctypes.data_as(C.POINTER(C.c_int64))))

    def _reduce_sa_call(self, text, stream):
        """csv_reduce_sa_device on a csv_sa_text: (sa_off address, filled csv_sa_cols)."""
        off_p, cols = C.POINTER(C.c_int64)(), _abi.csv_sa_cols()
        _lib.check(self.L.csv_reduce_sa_device(self.h, C.byref(text), C.c_void_p(stream or None), C.byref(off_p), C.byref(cols)))
        return off_p, cols

    def _reduce_packet_sa(self, d, stream):
        """A DevicePacket with SA text: its csv_read_cols::sa_off and csv_sa_cols become csv_reduce_sa_device's outputs."""
        if d.sa_text is None:
            return
        off_p, cols = self._reduce_sa_call(d.sa_text, stream)
        d[0].sa_off = off_p
        C.memmove(C.addressof(d[3]), C.addressof(cols), C.sizeof(cols))

    def reduce_sa(self, text, text_off, stream=None):
        """SA:Z values reduced on the device (csv_reduce_sa_device): text (uint8) and text_off (int64, n + 1) torch CUDA tensors, record
        i's value text[text_off[i]:text_off[i + 1]] without tag prefix or NUL, matched against set_contigs(..., names).  Returns
        zero-copy torch views (sa_off int64 [n + 1], dict of the seven int32 csv_sa_cols columns, _abi.SA_FIELDS), the sa_off / sa of
        a device packet.  They are library memory, valid until the next reduce_sa (or a packet with sa_text), set_contigs with names
        or close(), so clone() what you keep."""
        import torch
        to, n1 = _abi._cai_check("sa_text_off", text_off, ("<i8",), self.device)
        tp, nb = _abi._cai_check("sa_text", text, ("|u1", "<u1"), self.device)
        if n1 < 1:
            raise ValueError("sa_text_off needs n + 1 >= 1 entries")
        t = _abi.csv_sa_text(n1 - 1, nb, C.cast(C.c_void_p(to), C.POINTER(C.c_int64)), C.cast(C.c_void_p(tp), C.POINTER(C.c_uint8)))
        off_p, cols = self._reduce_sa_call(t, self._producer_stream(stream, [{"t": text, "o": text_off}]))
        dev = torch.device("cuda", self.device)
        off = torch.as_tensor(_DeviceView(C.cast(off_p, C.c_void_p).value, (n1,), "<i8"), device=dev)
        return off, {f: torch.as_tensor(_DeviceView(C.cast(getattr(cols, f), C.c_void_p).value, (cols.n,)), device=dev)
                     for f in _abi.SA_FIELDS}

    def fetch_alignments(self):
        """D2H of csv_cluster's alignment table (upload_alignments, or installed by rank_names after scan(..., alignments=True)):
        dict(chrom, start, end, read_id, is_primary) in the table's order, or None when there is none."""
        n = C.c_int64(0)
        rc = self.L.csv_fetch_alignments(self.h, C.c_int64(0), None, None, None, None, None, C.byref(n))
        if rc != _abi.CSV_E_CAPACITY:   # the size probe
            _lib.check(rc)
        if n.value == 0:
            return None
        k = n.value
        cols = {c: np.zeros(k, dtype=np.int32) for c in ("chrom", "start", "end", "read_id")}
        cols["is_primary"] = np.zeros(k, dtype=np.uint8)
        _lib.check(self.L.csv_fetch_alignments(self.h, C.c_int64(k), *[_abi.ptr(cols[c]) for c in ("chrom", "start", "end", "read_id")],
                                               cols["is_primary"].ctypes.data_as(C.POINTER(C.c_uint8)), C.byref(n)))
        return cols

    def scan(self, packet, alignments=False, stream=None):
        """Appends every decoded record of a BAM packet (csv_scan_append_named_device): a torch CUDA packet with names / name_off and
        no read_id (_abi.scan_packet).  The library drops what the reference's single_pipe drops (no CIGAR, contig < 0, flag 256 or
        272, outside the set_scan_regions table) and extracts the rest in place; alignments=True also keeps every record with a CIGAR
        and a contig as a row of the TRA genotyper's alignment table, which rank_names() installs.  Record numbers (provisional ids,
        name_rank_tensor, fetch_records, INS pieces) count all scanned records.  A packet may carry sa_text / sa_text_off instead of
        sa / sa_off, reduced on the device first as extract() does.  Returns extract()'s dict plus n_aln_rows."""
        d = _abi.scan_packet(packet, self.device)
        rc_, cig_p, n_cig, sa_, seq = d
        counts = (C.c_int64 * _abi.CSV_NTYPES)()
        n_rows, n_aln = C.c_int64(0), C.c_int64(0)
        st = self._producer_stream(stream, [packet])
        self._reduce_packet_sa(d, st)
        _lib.check(self.L.csv_scan_append_named_device(self.h, C.byref(rc_), cig_p, C.c_int64(n_cig), C.byref(sa_),
                                                       C.byref(seq) if seq is not None else None, C.byref(d.names), int(bool(alignments)),
                                                       C.c_void_p(st or None), counts, C.byref(n_rows), C.byref(n_aln)))
        out = self._extracted(counts, n_rows, True)
        out["n_aln_rows"] = int(n_aln.value)
        return out

    def fetch_ins_seqs(self, rows):
        """Sequence strings of INS rows `rows` from the device-built arena (csv_fetch_ins_seqs: one gather, one D2H copy).
        Needs an accumulation whose packets all were device packets with bases; CuteSVError CSV_E_STATE otherwise."""
        rows = np.ascontiguousarray(rows, dtype=np.int64).reshape(-1)
        whole, o = self._fetch_arena(self.L.csv_fetch_ins_seqs, rows.ctypes.data_as(C.POINTER(C.c_int64)), len(rows), 512 * len(rows) + 4096)
        whole = whole.decode("ascii")
        return [whole[o[i]:o[i + 1]] for i in range(len(rows))]

    def _fetch_arena(self, fn, rows, n, cap):
        """(bytes, offsets list) of csv_fetch_ins_seqs / csv_fetch_names on n rows: first with `cap` bytes of room, then with the
        room a CSV_E_CAPACITY reports."""
        off = np.zeros(n + 1, dtype=np.int64)
        while True:
            out = np.zeros(max(cap, 1), dtype=np.uint8)
            rc = fn(self.h, rows, C.c_int64(n), out.ctypes.data_as(C.POINTER(C.c_uint8)), C.c_int64(cap), off.ctypes.data_as(C.POINTER(C.c_int64)))
            if rc != _abi.CSV_E_CAPACITY:
                break
            cap = int(off[n])
        _lib.check(rc)
        return out[:int(off[n])].tobytes(), off.tolist()

    def ins_seq_tensors(self):
        """Zero-copy torch views of the device-built INS sequence arena: (bytes uint8, start int64 [n_rows], length int32 [n_rows]);
        row k's string is bytes[start[k]:start[k] + length[k]].  Valid until the next extract, upload or swap_ins_rows on this
        engine, so clone() whatever you keep."""
        import torch
        b, s, ln, nr = C.c_void_p(), C.c_void_p(), C.c_void_p(), C.c_int64(0)
        _lib.check(self.L.csv_ins_seq_device_ptrs(self.h, C.byref(b), C.byref(s), C.byref(ln), C.byref(nr)))
        dev = torch.device("cuda", self.device)
        n = nr.value
        start = torch.as_tensor(_DeviceView(s.value, (n,), "<i8"), device=dev)
        length = torch.as_tensor(_DeviceView(ln.value, (n,)), device=dev)
        nbytes = int((start + length.to(torch.int64)).max()) if n else 0
        return torch.as_tensor(_DeviceView(b.value, (nbytes,), "|u1"), device=dev), start, length

    def rank_names(self):
        """Ranks the read names of a named accumulation on the device (csv_rank_names): every signature's and reads row's read id
        becomes the dense rank of its name in byte (for UTF-8: Python str) order.  After scan(..., alignments=True) it also installs
        the scanned alignment rows, ids as ranks and sorted by contig, as the TRA genotyper's table.  Returns the number of distinct
        names."""
        nd = C.c_int64(0)
        _lib.check(self.L.csv_rank_names(self.h, C.byref(nd)))
        return int(nd.value)

    def fetch_names(self, ranks):
        """Read names (str) of name ranks `ranks` (any order, repeats allowed) after rank_names (csv_fetch_names)."""
        ranks = np.ascontiguousarray(ranks, dtype=np.int32).reshape(-1)
        raw, o = self._fetch_arena(self.L.csv_fetch_names, _abi.ptr(ranks), len(ranks), 64 * len(ranks) + 256)
        return [raw[o[i]:o[i + 1]].decode("utf-8") for i in range(len(ranks))]

    def name_rank_tensor(self):
        """Zero-copy torch view (int32, one entry per record of the accumulation) of the table record index -> name rank that
        rank_names built, e.g. to turn a caller-built alignment table's provisional ids into ranks with one gather.  Valid until the
        next extract or extract_reset on this engine, so clone() what you keep."""
        import torch
        p, nr = C.c_void_p(), C.c_int64(0)
        _lib.check(self.L.csv_name_ranks_device_ptr(self.h, C.byref(p), C.byref(nr)))
        return torch.as_tensor(_DeviceView(p.value, (nr.value,)), device=torch.device("cuda", self.device))

    def order_ins_ties(self):
        """Puts INS rows that tie on (contig, int(pos), len, read) into the order of their device-built sequences (csv_order_ins_ties):
        what ins_tie_swaps + swap_ins_rows do on the host.  The read ids must be ranks (rank_names or remap_read_ids first).  Returns
        the number of rows whose content moved."""
        nm = C.c_int64(0)
        _lib.check(self.L.csv_order_ins_ties(self.h, C.byref(nm)))
        return int(nm.value)

    def extract_skipped(self):
        """Records whose split-read analysis was skipped (more than 64 qualifying segments, only with max_split_parts -1)."""
        return int(self.L.csv_extract_skipped(self.h))

    def extract_reset(self):
        _lib.check(self.L.csv_extract_reset(self.h))
        self._ex_counts = [0] * _abi.CSV_NTYPES
        self._ex_rows = 0
        self._ex_pieces = 0
        self._ex_appending = False
        self._dev_rows = [0] * (_abi.CSV_NTYPES + 1)

    def fetch_ins_pieces(self, first_sig, n_sig, first_piece, n_piece):
        """Piece descriptors of INS signatures [first_sig, first_sig + n_sig) and pieces [first_piece, first_piece + n_piece):
        what the host needs to rebuild the sequences of the rows ONE packet appended.  piece_off is re-based to the slice."""
        po = np.zeros(max(n_sig, 1), dtype=np.int32)
        pc = np.zeros(max(n_sig, 1), dtype=np.int32)
        if n_sig:
            _lib.check(self.L.csv_fetch_sigs_range(self.h, _abi.CSV_INS, C.c_int64(first_sig), C.c_int64(n_sig), None, None, None, None, None,
                                                   _abi.ptr(po), _abi.ptr(pc)))
        pieces = np.zeros((max(n_piece, 1), 4), dtype=np.int32)
        if n_piece:
            _lib.check(self.L.csv_fetch_pieces_range(self.h, C.c_int64(first_piece), C.c_int64(n_piece), _abi.ptr(pieces)))
        return po[:n_sig] - first_piece, pc[:n_sig], pieces[:n_piece]

    def fetch_sig_cols(self, name, cols=("chrom", "a", "b", "read_id", "c")):
        """D2H of whole columns of the device-resident signatures of one type."""
        t = _abi.TYPE_IDS[name]
        k = self._ex_counts[t]
        out = {c: (np.zeros(max(k, 1), dtype=np.int32) if c in cols else None) for c in ("chrom", "a", "b", "read_id", "c")}
        if k:
            _lib.check(self.L.csv_fetch_sigs_range(self.h, t, C.c_int64(0), C.c_int64(k), *[(_abi.ptr(out[c]) if out[c] is not None else None)
                                                                                              for c in ("chrom", "a", "b", "read_id", "c")], None, None))
        return {c: (v[:k] if v is not None else None) for c, v in out.items()}

    def fetch_read_rows(self):
        """D2H of the device-resident reads table (reads_info_list rows, cuteSV:729-733)."""
        nr = self._ex_rows
        rows = {k: np.zeros(max(nr, 1), dtype=np.int32) for k in ("chrom", "start", "end", "read_id")}
        prim = np.zeros(max(nr, 1), dtype=np.uint8)
        _lib.check(self.L.csv_fetch_read_rows(self.h, C.c_int64(max(nr, 1)), _abi.ptr(rows["chrom"]), _abi.ptr(rows["start"]), _abi.ptr(rows["end"]),
                                              _abi.ptr(rows["read_id"]), prim.ctypes.data_as(C.POINTER(C.c_uint8))))
        rows = {k: v[:nr] for k, v in rows.items()}
        rows["is_primary"] = prim[:nr]
        return rows

    def remap_read_ids(self, rank):
        rank = np.ascontiguousarray(rank, dtype=np.int32)
        _lib.check(self.L.csv_remap_read_ids(self.h, _abi.ptr(rank), C.c_int64(len(rank))))

    def swap_ins_rows(self, pairs):
        pairs = np.ascontiguousarray(pairs, dtype=np.int64).reshape(-1, 2)
        if len(pairs):
            _lib.check(self.L.csv_swap_ins_rows(self.h, pairs.ctypes.data_as(C.POINTER(C.c_int64)), C.c_int64(len(pairs))))

    def fetch_extracted(self):
        """D2H of everything csv_extract produced (parity tests / host ALT strings)."""
        sigs = {}
        poff = pcnt = None
        for t, name in enumerate(_abi.TYPE_NAMES):
            k = self._ex_counts[t]
            cols = {c: np.zeros(max(k, 1), dtype=np.int32) for c in ("chrom", "a", "b", "read_id", "c")}
            po = np.zeros(max(k, 1), dtype=np.int32)
            pc = np.zeros(max(k, 1), dtype=np.int32)
            _lib.check(self.L.csv_fetch_sigs(self.h, t, C.c_int64(max(k, 1)), _abi.ptr(cols["chrom"]), _abi.ptr(cols["a"]), _abi.ptr(cols["b"]),
                                             _abi.ptr(cols["read_id"]), _abi.ptr(cols["c"]), _abi.ptr(po), _abi.ptr(pc)))
            sigs[name] = {c: v[:k] for c, v in cols.items()}
            if name == "INS":
                poff, pcnt = po[:k], pc[:k]
        npz = C.c_int64(0)
        _lib.check(self.L.csv_fetch_pieces(self.h, C.c_int64(0), None, C.byref(npz)))
        pieces = np.zeros((max(npz.value, 1), 4), dtype=np.int32)
        _lib.check(self.L.csv_fetch_pieces(self.h, C.c_int64(len(pieces)), _abi.ptr(pieces), C.byref(npz)))
        return dict(sigs=sigs, piece_off=poff, piece_cnt=pcnt, pieces=pieces[:npz.value], rows=self.fetch_read_rows())


class _DeviceView(object):
    """__cuda_array_interface__ of an array the library owns (torch.as_tensor makes a view of it, no copy); int32 by default."""

    def __init__(self, ptr, shape, typestr="<i4"):
        self.__cuda_array_interface__ = {"shape": tuple(shape), "typestr": typestr, "data": (int(ptr or 0), False), "version": 2}
