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

// RawRows is one row set of a flush as columns: n rawRows (lib/storage/raw_row.go:12), TSIDs marshaled (tsid.go:62).
type RawRows struct {
	TSIDs         []byte // n * 24
	Timestamps    []int64
	Values        []float64
	PrecisionBits []uint8
}

// PartsFromRows is rawRowsMarshaler.marshalToInmemoryPart (lib/storage/raw_row.go:81) for every set at once on the GPU: one part
// per set, an empty part for an empty set. Rows with equal (TSID, Timestamp) keep their input order. The ctx's dedup interval
// (SetDedupInterval) applies. The returned files are copies the caller owns.
func (c *Ctx) PartsFromRows(sets []RawRows) ([]PartFiles, []MergeStats, error) {
	if len(sets) == 0 {
		return nil, nil, nil
	}
	var pin runtime.Pinner
	defer pin.Unpin()
	rows := make([]C.vmb_raw_rows, len(sets))
	for i := range sets {
		s := &sets[i]
		r := &rows[i]
		n := len(s.Timestamps)
		if n > 0 {
			pin.Pin(&s.TSIDs[0])
			pin.Pin(&s.Timestamps[0])
			pin.Pin(&s.Values[0])
			pin.Pin(&s.PrecisionBits[0])
			r.tsids = (*C.uint8_t)(unsafe.Pointer(&s.TSIDs[0]))
			r.timestamps = (*C.int64_t)(unsafe.Pointer(&s.Timestamps[0]))
			r.values = (*C.double)(unsafe.Pointer(&s.Values[0]))
			r.precision_bits = (*C.uint8_t)(unsafe.Pointer(&s.PrecisionBits[0]))
		}
		r.n = C.uint64_t(n)
	}
	mps := make([]*C.vmb_merged_part, len(sets))
	sts := make([]C.vmb_merge_stats, len(sets))
	if rc := C.vmb_parts_from_rows(c.p, &rows[0], C.size_t(len(sets)), &mps[0], &sts[0]); rc != 0 {
		return nil, nil, lastError(rc, "vmb_parts_from_rows")
	}
	parts := make([]PartFiles, len(sets))
	stats := make([]MergeStats, len(sets))
	cp := func(p *C.uint8_t, n C.uint64_t) []byte { return C.GoBytes(unsafe.Pointer(p), C.int(n)) }
	for i, mp := range mps {
		var out C.vmb_part_files
		C.vmb_merged_part_files(mp, &out)
		parts[i] = PartFiles{
			Metaindex:  cp(out.metaindex, out.metaindex_len),
			Index:      cp(out.index, out.index_len),
			Timestamps: cp(out.timestamps, out.timestamps_len),
			Values:     cp(out.values, out.values_len),
		}
		st := &sts[i]
		stats[i] = MergeStats{uint64(st.rows_count), uint64(st.blocks_count), int64(st.min_ts), int64(st.max_ts),
			uint64(st.rows_merged), uint64(st.rows_deleted)}
		C.vmb_merged_part_free(mp)
	}
	return parts, stats, nil
}
