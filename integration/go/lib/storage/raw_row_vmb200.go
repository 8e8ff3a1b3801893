//go:build cgo && vmb200

package storage

import (
	"github.com/VictoriaMetrics/VictoriaMetrics/lib/vmb200"
)

// flushRowssVMB200 is what flushRowssToInmemoryParts (partition.go:603) becomes: every shard's rows turn into parts in one
// library call (in place of createInmemoryPart per shard, :880), and those parts are merged by one more call (in place of
// mustMergeInmemoryParts). The caller wraps the merged files as an in-memory part with ph and hands it to addToInmemoryParts,
// as before; a part above getMaxInmemoryPartSize() is kept apart the same way.
func flushRowssVMB200(ph *partHeader, rowss [][]rawRow, retentionDeadline int64) (vmb200.PartFiles, error) {
	sets := make([]vmb200.RawRows, 0, len(rowss))
	for _, rows := range rowss {
		s := vmb200.RawRows{
			TSIDs:         make([]byte, 0, 24*len(rows)),
			Timestamps:    make([]int64, len(rows)),
			Values:        make([]float64, len(rows)),
			PrecisionBits: make([]uint8, len(rows)),
		}
		for i := range rows {
			r := &rows[i]
			s.TSIDs = r.TSID.Marshal(s.TSIDs)
			s.Timestamps[i], s.Values[i], s.PrecisionBits[i] = r.Timestamp, r.Value, r.PrecisionBits
		}
		sets = append(sets, s)
	}
	c := vmb200.Get()
	defer vmb200.Put(c)
	c.SetDedupInterval(GetDedupInterval())
	parts, _, err := c.PartsFromRows(sets)
	if err != nil {
		return vmb200.PartFiles{}, err
	}
	out, st, err := c.MergeParts(parts, retentionDeadline, nil)
	if err != nil {
		return vmb200.PartFiles{}, err
	}
	ph.Reset()
	ph.RowsCount, ph.BlocksCount = st.RowsCount, st.BlocksCount
	ph.MinTimestamp, ph.MaxTimestamp = st.MinTimestamp, st.MaxTimestamp
	return out, nil
}
