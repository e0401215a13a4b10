// NOT COMPILED OR RUN IN THIS REPOSITORY'S ENVIRONMENT (no Go toolchain): see bestfit.go.
package bestfit

import "testing"

const capMem = 183359 // MiB per card of the synthetic node (elastic-gpu-agent_b200/synth.py)

func fullTable() ([]int32, []int32) {
	fc, fm := make([]int32, 8), make([]int32, 8)
	for d := range fc {
		fc[d], fm[d] = 100, capMem
	}
	return fc, fm
}

// cfg1 known answers (SURVEY.md Appendix A.6, tests/golden/bestfit_kat.json).
func TestCfg1(t *testing.T) {
	fc, fm := fullTable()
	core := []int32{25, 25, 25, 25, 25}
	mem := []int32{1024, 1024, 1024, 1024, 1024}
	idx := make([]int32, 5)
	dc, _ := Snapshot(fc, fm, core, mem, idx)
	for _, d := range idx {
		if d != 0 {
			t.Fatalf("snapshot: want all 0, got %v", idx)
		}
	}
	if dc[0] != 125 {
		t.Fatalf("snapshot demand: want 125, got %d", dc[0])
	}
	Sequential(fc, fm, core, mem, idx)
	want := []int32{0, 0, 0, 0, 1}
	for i := range want {
		if idx[i] != want[i] {
			t.Fatalf("sequential: want %v, got %v", want, idx)
		}
	}
	if fc[0] != 0 || fc[1] != 75 || fm[0] != capMem-4096 {
		t.Fatalf("sequential table: %v %v", fc, fm)
	}
	if Pick(fc, fm, 101, 1) != -1 {
		t.Fatal("core 101 must be infeasible")
	}
}

// splitmix64 of the repo's counter-based generator (elastic-gpu-agent_b200/synth.py), reduced
// to what a benchmark needs: any fixed pseudo-random requests will do here.
func splitmix64(x uint64) uint64 {
	x += 0x9E3779B97F4A7C15
	x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9
	x = (x ^ (x >> 27)) * 0x94D049BB133111EB
	return x ^ (x >> 31)
}

func BenchmarkSnapshot1M(b *testing.B) {
	const rows = 1 << 20
	fc := []int32{2, 98, 60, 61, 86, 23, 5, 90}
	fm := []int32{90000, 1200, 183000, 52000, 7000, 140000, 66000, 31000}
	core, mem, idx := make([]int32, rows), make([]int32, rows), make([]int32, rows)
	for i := range core {
		core[i] = int32(1 + splitmix64(uint64(i))%100)
		mem[i] = int32(1 + splitmix64(uint64(i)+rows)%65536)
	}
	b.SetBytes(12 * rows)
	b.ResetTimer()
	for n := 0; n < b.N; n++ {
		Snapshot(fc, fm, core, mem, idx)
	}
	// SetBytes makes `go test -bench` print MB/s of algorithmic traffic; decisions/s = that / 12 B
}
