//go:build cgo && vmb200

package storage

import (
	"sync/atomic"

	"github.com/VictoriaMetrics/VictoriaMetrics/lib/uint64set"
	"github.com/VictoriaMetrics/VictoriaMetrics/lib/vmb200"
)

// mergePartsVMB200 is what mergeBlockStreams (merge.go:19) becomes at its call site (partition.go:1606) when the parts' files
// are in memory: one library call that returns the merged part's four files and its partHeader. The caller still writes the
// files under their names (part.go:34), metadata.json with MinDedupInterval, and keeps stopCh: a started GPU merge runs to its end.
func mergePartsVMB200(ph *partHeader, parts []vmb200.PartFiles, dmis *uint64set.Set, retentionDeadline int64,
	rowsMerged, rowsDeleted *atomic.Uint64) (vmb200.PartFiles, error) {
	c := vmb200.Get()
	defer vmb200.Put(c)
	c.SetDedupInterval(GetDedupInterval())
	out, st, err := c.MergeParts(parts, retentionDeadline, dmis.AppendTo(nil)) // AppendTo returns the ids sorted
	if err != nil {
		return vmb200.PartFiles{}, err
	}
	ph.Reset()
	ph.RowsCount, ph.BlocksCount = st.RowsCount, st.BlocksCount
	ph.MinTimestamp, ph.MaxTimestamp = st.MinTimestamp, st.MaxTimestamp
	rowsMerged.Add(st.RowsMerged)
	rowsDeleted.Add(st.RowsDeleted)
	return out, nil
}
