//go:build cgo && vmb200

package vmb200

/*
#include <stdlib.h>
#include "vmb200.h"
*/
import "C"

import (
	"runtime"
	"unsafe"
)

// PartFiles holds the four data files of a part (lib/storage/part.go:34).
type PartFiles struct {
	Metaindex, Index, Timestamps, Values []byte
}

// MergeStats is the partHeader of the merged part and the counters mergeBlockStreams updates.
type MergeStats struct {
	RowsCount, BlocksCount     uint64
	MinTimestamp, MaxTimestamp int64
	RowsMerged, RowsDeleted    uint64
}

// MergeParts is mergeBlockStreams (lib/storage/merge.go:19) over parts, in the order of the blockStreamReaders, on the GPU.
// dmis holds the deleted MetricIDs sorted ascending; the ctx's dedup interval (SetDedupInterval) applies. The returned files are
// copies the caller owns.
func (c *Ctx) MergeParts(parts []PartFiles, retentionDeadline int64, dmis []uint64) (PartFiles, MergeStats, error) {
	// files holds pointers into the parts' slices: pin them for the call (cgo pointer rules)
	var pin runtime.Pinner
	defer pin.Unpin()
	files := make([]C.vmb_part_files, len(parts))
	for i := range parts {
		p := &parts[i]
		f := &files[i]
		for _, b := range [][]byte{p.Metaindex, p.Index, p.Timestamps, p.Values} {
			if len(b) > 0 {
				pin.Pin(&b[0])
			}
		}
		f.metaindex, f.metaindex_len = bytePtr(p.Metaindex), C.uint64_t(len(p.Metaindex))
		f.index, f.index_len = bytePtr(p.Index), C.uint64_t(len(p.Index))
		f.timestamps, f.timestamps_len = bytePtr(p.Timestamps), C.uint64_t(len(p.Timestamps))
		f.values, f.values_len = bytePtr(p.Values), C.uint64_t(len(p.Values))
	}
	var fp *C.vmb_part_files
	if len(files) > 0 {
		fp = &files[0]
	}
	var dp *C.uint64_t
	if len(dmis) > 0 {
		dp = (*C.uint64_t)(unsafe.Pointer(&dmis[0]))
	}
	var mp *C.vmb_merged_part
	var st C.vmb_merge_stats
	if rc := C.vmb_merge_parts(c.p, fp, C.size_t(len(parts)), C.int64_t(retentionDeadline), dp, C.size_t(len(dmis)), &mp, &st); rc != 0 {
		return PartFiles{}, MergeStats{}, lastError(rc, "vmb_merge_parts")
	}
	defer C.vmb_merged_part_free(mp)
	var out C.vmb_part_files
	C.vmb_merged_part_files(mp, &out)
	cp := func(p *C.uint8_t, n C.uint64_t) []byte { return C.GoBytes(unsafe.Pointer(p), C.int(n)) }
	res := PartFiles{
		Metaindex:  cp(out.metaindex, out.metaindex_len),
		Index:      cp(out.index, out.index_len),
		Timestamps: cp(out.timestamps, out.timestamps_len),
		Values:     cp(out.values, out.values_len),
	}
	return res, MergeStats{uint64(st.rows_count), uint64(st.blocks_count), int64(st.min_ts), int64(st.max_ts),
		uint64(st.rows_merged), uint64(st.rows_deleted)}, nil
}
